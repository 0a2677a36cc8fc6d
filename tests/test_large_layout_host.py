"""The slab layout at its documented limits, without a GPU (layout-only plans, device=-1): one tensor of 2^32 - 1
elements, a slab of exactly 2^37 elements, and the data-parallel shard arithmetic on a layout whose tiles and slab
offsets pass 2^31 (include/gaccum.h, gaccum_plan_create).

Every expected value is computed here in Python integers from the layout rules alone: tensors start at multiples of 32
elements, each is cut into tiles of 2048 from its start, and shard boundary r is the first tile whose cumulative
element count reaches ceil(r * P / world).  Each 2^37-element layout builds a tile table of ~2^26 entries (1 GB of host
memory, about a second).
"""
import numpy as np
import pytest

import gaccum_b200 as g
from gaccum_b200 import _lib

TILE = 2048
ALIGN = 32
BIG = 2 ** 31 + 6151
DP_LAYOUT = (1000, BIG, 5, 33)


def _tiles(n: int) -> int:
    return -(-n // TILE)


def _padded(n: int) -> int:
    return -(-n // ALIGN) * ALIGN


class Layout:
    """The plan's layout restated: offsets, tile counts and the shard rule of gaccum_abi.cu, per tensor (no per-tile
    arrays, so it stays cheap at 2^26 tiles)."""

    def __init__(self, numels):
        self.numels = [int(n) for n in numels]
        self.offsets, self.first_tile, self.before = [], [], []      # slab offset, global index of tile 0, elements before
        off = t = c = 0
        for n in self.numels:
            self.offsets.append(off); self.first_tile.append(t); self.before.append(c)
            off += _padded(n); t += _tiles(n); c += n
        self.padded, self.num_tiles, self.P = off, t, c

    def _tensor_of(self, t: int) -> int:
        for i in range(len(self.numels) - 1, -1, -1):
            if self.first_tile[i] <= t and _tiles(self.numels[i]) > 0:
                return i
        raise AssertionError(t)

    def slab_offset(self, t: int) -> int:
        """Where tile t starts in the slab; the slab's end for t == num_tiles."""
        if t == self.num_tiles:
            return self.padded
        i = self._tensor_of(t)
        return self.offsets[i] + (t - self.first_tile[i]) * TILE

    def cumulative(self, t: int) -> int:
        """Elements in tiles [0, t)."""
        if t == self.num_tiles:
            return self.P
        i = self._tensor_of(t)
        return self.before[i] + (t - self.first_tile[i]) * TILE

    def bounds(self, world: int):
        """gaccum_abi.cu shard_bounds: bounds[r] = 1 + the first tile whose cumulative count reaches
        ceil(r * P / world), for 0 < r < world."""
        out = [0]
        for r in range(1, world):
            target = (self.P * r + world - 1) // world
            for i, n in enumerate(self.numels):
                if n and self.before[i] + n >= target:
                    out.append(self.first_tile[i] + max(1, -(-(target - self.before[i]) // TILE)))
                    break
        out.append(self.num_tiles)
        return out

    def stage_elements(self, world: int) -> int:
        b = self.bounds(world)
        span = max(self.slab_offset(b[r + 1]) - self.slab_offset(b[r]) for r in range(world))
        return max(span, ALIGN) * (world - 1)


def _plan(numels, hp=None):
    return g.Plan(list(numels), None, hp or g.HParams.bert(), device=-1)


def _refused(numels, message: str):
    with pytest.raises(g.GaccumError) as e:
        _plan(numels)
    assert e.value.code == _lib.EINVAL and message in str(e.value), str(e.value)


# ---- one tensor of 2^32 - 1 elements --------------------------------------------------------------------------------------
@pytest.mark.parametrize("hp, apply_bytes", [(g.HParams.bert(), 36), (g.HParams.tf_adam(), 36), (g.HParams.lamb(), 48)])
def test_largest_tensor(hp, apply_bytes):
    n = 2 ** 32 - 1
    plan = _plan([n], hp)
    assert plan.num_tiles == 2 ** 21
    assert plan.offsets == [0] and plan.padded_size == 2 ** 32
    assert plan.num_elements == n
    assert plan.algorithmic_bytes(True) == apply_bytes * n and plan.algorithmic_bytes(False) == 12 * n
    assert plan.algorithmic_bytes(True) > 2 ** 32           # int64 all the way: 36 x (2^32 - 1) does not fit 32 bits


def test_tensor_of_2_32_elements_is_refused():
    _refused([2 ** 32], "limit is 2^32-1")
    _refused([5, 2 ** 32, 7], "limit is 2^32-1")


def test_tensors_past_2_32_elements_in_total():
    """Two tensors of 2^32 - 1: the second starts at slab offset 2^32, past every 32-bit element offset."""
    n = 2 ** 32 - 1
    plan = _plan([n, 3, n])
    lay = Layout([n, 3, n])
    assert plan.offsets == lay.offsets == [0, 2 ** 32, 2 ** 32 + 32]
    assert plan.padded_size == 2 ** 33 + 32 and plan.num_elements == 2 * n + 3
    assert plan.num_tiles == 2 ** 22 + 1


# ---- a slab of 2^37 elements ----------------------------------------------------------------------------------------------
LIMIT = [2 ** 32 - 1] * 32                  # each padded to 2^32: exactly 2^37
# also exactly 2^37, with a thousand 1-element tensors (31 elements of padding each) at the end: the last data-parallel
# shard spans the most slab for the elements it holds
LIMIT_TAIL = [2 ** 32 - 1] * 31 + [2 ** 32 - 32000] + [1] * 1000
LIMITS = {"equal": LIMIT, "tail": LIMIT_TAIL}


@pytest.fixture(scope="module", params=sorted(LIMITS))
def limit(request):
    numels = LIMITS[request.param]
    plan = _plan(numels)
    yield plan, Layout(numels)
    plan.close()


def test_slab_of_2_37_elements_is_accepted(limit):
    plan, lay = limit
    assert plan.padded_size == lay.padded == 2 ** 37
    assert plan.offsets == lay.offsets and plan.offsets[31] == 31 * 2 ** 32
    assert plan.num_elements == lay.P and plan.num_tiles == lay.num_tiles
    assert plan.algorithmic_bytes(True) == 36 * lay.P and plan.algorithmic_bytes(False) == 12 * lay.P


def test_slab_of_2_37_tile_count():
    plan = _plan(LIMIT)
    assert plan.num_tiles == 2 ** 26 and plan.num_elements == 32 * (2 ** 32 - 1)


@pytest.mark.parametrize("world", [2, 3, 5, 8])
def test_stage_elements_at_2_37(limit, world):
    """The last shard of a 2^37-element slab ends at slab offset 2^37, 2^32 in units of 32: its span must not wrap (to a
    negative span, which would size the staging area by the other shards alone)."""
    plan, lay = limit
    assert plan.dp_stage_elements(world) == lay.stage_elements(world)
    b = lay.bounds(world)
    for r in range(world):
        assert plan.dp_shard_range(world, r) == (b[r], b[r + 1], lay.cumulative(b[r + 1]) - lay.cumulative(b[r]))


def test_zero_element_tensor_at_2_37_is_accepted():
    plan = _plan(LIMIT + [0])
    assert plan.offsets[-1] == 2 ** 37 and plan.padded_size == 2 ** 37 and plan.num_tiles == 2 ** 26


def test_one_element_past_2_37_is_refused():
    _refused(LIMIT + [1], "slab too large")


def test_padding_past_2_37_is_refused():
    """Every tile of these layouts starts below 2^37 (its last one at 2^37 - 32), but the padded slab ends 2016 and 32
    elements past it."""
    _refused([2016] + LIMIT, "slab too large")
    _refused([2 ** 32 - 1] * 31 + [2 ** 32 - 2080, TILE + 64], "slab too large")


# ---- data-parallel shards past 2^31 ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_dp_shards_past_2_31(world):
    plan = _plan(DP_LAYOUT)
    lay = Layout(DP_LAYOUT)
    assert plan.offsets == lay.offsets and plan.num_tiles == lay.num_tiles and plan.padded_size == lay.padded
    b = lay.bounds(world)
    total = np.int64(0)
    prev_hi = 0
    for r in range(world):
        lo, hi, n = plan.dp_shard_range(world, r)
        assert lo == prev_hi, "shards must tile the layout without gap or overlap"
        assert (lo, hi) == (b[r], b[r + 1])
        assert n == lay.cumulative(hi) - lay.cumulative(lo)
        # every shard starts at a tile start: slab offset = its tensor's offset + a multiple of 2048
        start = lay.slab_offset(lo)
        if lo < lay.num_tiles:
            i = lay._tensor_of(lo)
            assert (start - lay.offsets[i]) % TILE == 0
        total += np.int64(n)
        prev_hi = hi
    assert prev_hi == plan.num_tiles and int(total) == plan.num_elements == sum(DP_LAYOUT)
    assert plan.dp_stage_elements(world) == lay.stage_elements(world)
    assert plan.dp_stage_elements(world) > 2 ** 31 // world
