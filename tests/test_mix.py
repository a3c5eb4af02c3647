"""The conference mixer on the CPU: the host build of its source (tests/hostsim/mix.cpp: sb_mix.cuh compiled by g++, in the
order of the two mix kernels) against a plain numpy restatement of the rule in include/solo_b200.h, at 0 tolerance.

Rooms of 0, 1, 2, k, k + 1, 33 and 1 000 members, listed out of order, for every k from 1 to 8; equal levels (tie order);
rooms with no eligible member; full-scale rows of one sign (saturation); 20 ms flags (bit 0 only)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "hostsim", "mix.cpp")
POISON = -21846                                 # 0xAAAA: rows of streams in no room must keep it


def load_lib(out):
    """Compile tests/hostsim/mix.cpp to `out` and load it."""
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-w", SRC, "-o", out])
    lib = C.CDLL(out)
    lib.mix_model.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int] + [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def L(tmp_path_factory):
    return load_lib(str(tmp_path_factory.mktemp("mix") / "libmix.so"))


def csr(rooms):
    room_start = np.zeros(len(rooms) + 1, np.int32)
    room_start[1:] = np.cumsum([len(r) for r in rooms])
    members = np.concatenate([np.asarray(r, np.int32) for r in rooms] + [np.zeros(0, np.int32)])
    return room_start, members


def numpy_mix(pcm, level, flags, rooms, k, out):
    """The rule of include/solo_b200.h, restated: sort each room's eligible members by (level, index), keep k, and give
    every member the clamped int32 sum of the kept rows minus its own."""
    talkers = np.full((len(rooms), k), -1, np.int32)
    for r, mem in enumerate(rooms):
        el = sorted((int(level[j]), int(j)) for j in mem if flags[j] & 3)[:k]
        t = [j for _, j in el]
        talkers[r, :len(t)] = t
        total = pcm[t].astype(np.int32).sum(0) if t else np.zeros(pcm.shape[1], np.int32)
        for i in mem:
            own = pcm[i].astype(np.int32) if int(i) in t else 0
            out[i] = np.clip(total - own, -32768, 32767).astype(np.int16)
    return out, talkers


def model_mix(L, pcm, level, flags, rooms, k, out):
    room_start, members = csr(rooms)
    talkers = np.full((len(rooms), k), 12345, np.int32)
    n, spp = pcm.shape
    L.mix_model(pcm.ctypes.data, out.ctypes.data, spp, n, level.ctypes.data, flags.ctypes.data, room_start.ctypes.data,
                members.ctypes.data, len(rooms), k, talkers.ctypes.data)
    return out, talkers


def layout(k, rng, sizes=None, spare=40):
    """Rooms of the given sizes (default 0, 1, 2, k, k + 1, 33, 1000) over a random permutation of the streams, in shuffled
    room order, and `spare` streams in no room; returns (n, rooms)."""
    sizes = list(sizes if sizes is not None else (0, 1, 2, k, k + 1, 33, 1000))
    rng.shuffle(sizes)
    n = sum(sizes) + spare
    perm = rng.permutation(n).astype(np.int32)
    rooms, o = [], 0
    for s in sizes:
        rooms.append(perm[o:o + s])
        o += s
    return n, rooms


def check(L, pcm, level, flags, rooms, k):
    n, spp = pcm.shape
    want, wt = numpy_mix(pcm, level, flags, rooms, k, np.full((n, spp), POISON, np.int16))
    got, gt = model_mix(L, pcm, level, flags, rooms, k, np.full((n, spp), POISON, np.int16))
    assert np.array_equal(gt, wt)
    assert np.array_equal(got, want)
    return wt


@pytest.mark.parametrize("k", range(1, 9))
def test_room_sizes_and_every_k(L, k):
    """Random rows, levels and flags (a third of the streams ineligible) at spp 640 and 1280."""
    rng = np.random.Generator(np.random.PCG64(100 + k))
    for spp in (640, 1280):
        n, rooms = layout(k, rng)
        pcm = rng.integers(-12000, 12000, (n, spp), dtype=np.int16)
        level = rng.integers(0, 128, n, dtype=np.uint8)
        flags = rng.choice(np.array([0, 1, 2, 3, 4, 8, 12, 5], np.uint8), n)
        t = check(L, pcm, level, flags, rooms, k)
        assert (t >= 0).sum() > 0 and (t < 0).sum() > 0


@pytest.mark.parametrize("k", (1, 3, 8))
def test_equal_levels_go_to_the_lower_index(L, k):
    """Every stream at the same level (and a second case with two levels): the talkers are the lowest eligible indices."""
    rng = np.random.Generator(np.random.PCG64(7 + k))
    n, rooms = layout(k, rng)
    pcm = rng.integers(-3000, 3000, (n, 640), dtype=np.int16)
    flags = np.full(n, 3, np.uint8)
    t = check(L, pcm, np.full(n, 40, np.uint8), flags, rooms, k)
    for r, mem in enumerate(rooms):
        assert list(t[r, :min(k, len(mem))]) == sorted(int(j) for j in mem)[:k]
    check(L, pcm, (np.arange(n) % 2 * 30).astype(np.uint8), flags, rooms, k)


def test_rooms_without_eligible_members_give_zeros(L):
    """Rooms whose members all report flags 0 or concealment only: no talkers, every member row zero."""
    rng = np.random.Generator(np.random.PCG64(3))
    n, rooms = layout(3, rng)
    pcm = rng.integers(-20000, 20000, (n, 640), dtype=np.int16)
    flags = rng.choice(np.array([0, 4, 8, 12], np.uint8), n)
    t = check(L, pcm, np.zeros(n, np.uint8), flags, rooms, 3)
    assert (t == -1).all()


@pytest.mark.parametrize("sign", (1, -1))
def test_full_scale_rows_saturate(L, sign):
    """Eight talkers of full-scale rows of one sign: every listener's sum clamps at 32767 / -32768, a talker's too."""
    rng = np.random.Generator(np.random.PCG64(11))
    n, rooms = layout(8, rng)
    full = 32767 if sign > 0 else -32768
    pcm = np.full((n, 640), full, np.int16)
    pcm[:, ::7] = sign * 30000
    level = rng.integers(0, 128, n, dtype=np.uint8)
    check(L, pcm, level, np.full(n, 3, np.uint8), rooms, 8)
    got, _ = model_mix(L, pcm, level, np.full(n, 3, np.uint8), rooms, 8, np.zeros((n, 640), np.int16))
    for mem in rooms:
        if len(mem) >= 3:                       # every member hears at least two full-scale rows
            assert (got[mem] == full).all()


def test_20ms_flags(L):
    """20 ms decoder rows (320 samples) whose flags use bit 0 only (bit 2 for a concealed frame)."""
    rng = np.random.Generator(np.random.PCG64(20))
    for k in (2, 5):
        n, rooms = layout(k, rng)
        pcm = rng.integers(-9000, 9000, (n, 320), dtype=np.int16)
        flags = rng.choice(np.array([0, 1, 4], np.uint8), n)
        t = check(L, pcm, rng.integers(0, 128, n, dtype=np.uint8), flags, rooms, k)
        assert all(flags[j] == 1 for j in t.ravel() if j >= 0)
