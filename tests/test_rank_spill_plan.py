"""CPU pin of hm_rank_spill_plan, the device plan of a rank's parked routed rounds when its lists are in host memory
(DESIGN.md §4c, *Lists in host memory*): it stays within the room and grows with it, keeps the caps, refuses below
the minimum with the sizes, and listing and more ranks need more per slot."""
import ctypes as C

import pytest

from smudgeplot_b200 import _lib


def plan(nc, ns, k, world, listing, room):
    lay = _lib.SpillLayout()
    rc = _lib.lib().hm_rank_spill_plan(nc, ns, k, world, listing, room, C.byref(lay))
    return rc, lay


@pytest.mark.parametrize("k", [21, 31, 32, 33, 64])
@pytest.mark.parametrize("world", [1, 2, 3, 8])
@pytest.mark.parametrize("listing", [0, 1])
def test_within_the_room_and_monotone(k, world, listing):
    last = (0, 0)
    for room in [1 << 22, 1 << 24, 1 << 26, 1 << 28, 1 << 30]:
        rc, lay = plan(10 ** 8, 10 ** 8, k, world, listing, room)
        assert rc == 0
        assert lay.slice_bytes + lay.part_bytes <= room
        assert lay.queries == 2 * lay.slice and lay.slice >= 1024 and lay.part >= 1024
        assert lay.slice >= last[0]
        last = (lay.slice, lay.part)


def test_everything_at_full_size_when_it_fits():
    rc, lay = plan(5000, 7000, 31, 2, 0, 1 << 30)
    assert rc == 0 and lay.slice == 5000 and lay.part == 7000


def test_caps():
    for world in (1, 3, 16):
        rc, lay = plan(1 << 40, 1 << 40, 31, world, 0, 1 << 62)
        assert rc == 0
        assert lay.slice <= _lib.SPILL_MAX_SLICE // world
        assert lay.part <= _lib.SPILL_MAX_PART


def test_refusal_names_the_sizes():
    rc, lay = plan(10 ** 6, 10 ** 6, 31, 2, 1, 1 << 16)
    assert rc == -3
    msg = _lib.lib().hm_last_error().decode()
    assert "65536 bytes of device room" in msg and "1024 candidates" in msg and "1024 S" in msg


def test_listing_needs_more_per_slot_and_the_receive_side_grows_with_the_ranks():
    room = 1 << 24
    c = plan(10 ** 8, 10 ** 8, 31, 2, 0, room)[1].slice
    lst = plan(10 ** 8, 10 ** 8, 31, 2, 1, room)[1].slice
    assert lst < c
    slices = [plan(10 ** 8, 10 ** 8, 31, w, 0, room)[1].slice for w in (1, 2, 4, 8)]
    assert slices == sorted(slices, reverse=True) and slices[0] > slices[-1]
    bytes_ = [plan(4096, 4096, 31, w, 0, 1 << 30)[1].slice_bytes for w in (1, 2, 4, 8)]
    assert bytes_ == sorted(bytes_) and bytes_[0] < bytes_[-1]


def test_bad_arguments():
    assert plan(-1, 0, 31, 1, 0, 1 << 20)[0] == -1
    assert plan(0, 0, 31, 0, 0, 1 << 20)[0] == -1
    assert plan(0, 0, 31, 17, 0, 1 << 20)[0] == -1
