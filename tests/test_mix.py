"""The conference mixer on the CPU: the host build of its source (tests/hostsim/server.cpp driven by sim.mix_model:
sb_mix.cuh compiled by g++, in the order of the two mix kernels) against a plain numpy restatement of the rule in
include/solo_b200.h (tests/server_ref.numpy_mix), at 0 tolerance.

Rooms of 0, 1, 2, k, k + 1, 33 and 1 000 members, listed out of order, for every k from 1 to 8; equal levels (tie order);
rooms with no eligible member; full-scale rows of one sign (saturation); 20 ms flags (bit 0 only)."""
import numpy as np
import pytest

from tests.parity import sim  # noqa: F401  (fixture)
from tests.server_ref import POISON, csr, numpy_mix, shuffled_rooms


def check(sim, pcm, level, flags, rooms, k):
    n, spp = pcm.shape
    want, wt = numpy_mix(pcm, level, flags, rooms, k, np.full((n, spp), POISON, np.int16))
    got, gt = sim.mix_model(pcm, level, flags, *csr(rooms), k, np.full((n, spp), POISON, np.int16))
    assert np.array_equal(gt, wt)
    assert np.array_equal(got, want)
    return wt


@pytest.mark.parametrize("k", range(1, 9))
def test_room_sizes_and_every_k(sim, k):
    """Random rows, levels and flags (a third of the streams ineligible) at spp 640 and 1280."""
    rng = np.random.Generator(np.random.PCG64(100 + k))
    for spp in (640, 1280):
        n, rooms = shuffled_rooms(k, rng)
        pcm = rng.integers(-12000, 12000, (n, spp), dtype=np.int16)
        level = rng.integers(0, 128, n, dtype=np.uint8)
        flags = rng.choice(np.array([0, 1, 2, 3, 4, 8, 12, 5], np.uint8), n)
        t = check(sim, pcm, level, flags, rooms, k)
        assert (t >= 0).sum() > 0 and (t < 0).sum() > 0


@pytest.mark.parametrize("k", (1, 3, 8))
def test_equal_levels_go_to_the_lower_index(sim, k):
    """Every stream at the same level (and a second case with two levels): the talkers are the lowest eligible indices."""
    rng = np.random.Generator(np.random.PCG64(7 + k))
    n, rooms = shuffled_rooms(k, rng)
    pcm = rng.integers(-3000, 3000, (n, 640), dtype=np.int16)
    flags = np.full(n, 3, np.uint8)
    t = check(sim, pcm, np.full(n, 40, np.uint8), flags, rooms, k)
    for r, mem in enumerate(rooms):
        assert list(t[r, :min(k, len(mem))]) == sorted(int(j) for j in mem)[:k]
    check(sim, pcm, (np.arange(n) % 2 * 30).astype(np.uint8), flags, rooms, k)


def test_rooms_without_eligible_members_give_zeros(sim):
    """Rooms whose members all report flags 0 or concealment only: no talkers, every member row zero."""
    rng = np.random.Generator(np.random.PCG64(3))
    n, rooms = shuffled_rooms(3, rng)
    pcm = rng.integers(-20000, 20000, (n, 640), dtype=np.int16)
    flags = rng.choice(np.array([0, 4, 8, 12], np.uint8), n)
    t = check(sim, pcm, np.zeros(n, np.uint8), flags, rooms, 3)
    assert (t == -1).all()


@pytest.mark.parametrize("sign", (1, -1))
def test_full_scale_rows_saturate(sim, sign):
    """Eight talkers of full-scale rows of one sign: every listener's sum clamps at 32767 / -32768, a talker's too."""
    rng = np.random.Generator(np.random.PCG64(11))
    n, rooms = shuffled_rooms(8, rng)
    full = 32767 if sign > 0 else -32768
    pcm = np.full((n, 640), full, np.int16)
    pcm[:, ::7] = sign * 30000
    level = rng.integers(0, 128, n, dtype=np.uint8)
    check(sim, pcm, level, np.full(n, 3, np.uint8), rooms, 8)
    got, _ = sim.mix_model(pcm, level, np.full(n, 3, np.uint8), *csr(rooms), 8, np.zeros((n, 640), np.int16))
    for mem in rooms:
        if len(mem) >= 3:                       # every member hears at least two full-scale rows
            assert (got[mem] == full).all()


def test_20ms_flags(sim):
    """20 ms decoder rows (320 samples) whose flags use bit 0 only (bit 2 for a concealed frame)."""
    rng = np.random.Generator(np.random.PCG64(20))
    for k in (2, 5):
        n, rooms = shuffled_rooms(k, rng)
        pcm = rng.integers(-9000, 9000, (n, 320), dtype=np.int16)
        flags = rng.choice(np.array([0, 1, 4], np.uint8), n)
        t = check(sim, pcm, rng.integers(0, 128, n, dtype=np.uint8), flags, rooms, k)
        assert all(flags[j] == 1 for j in t.ravel() if j >= 0)
