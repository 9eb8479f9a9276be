"""The field pool's slot policies (csrc/pfnav_pool_host.h, compiled with g++ through tests/emu/pool_emu.cpp) on random
sequences of reservations with random touch stamps, zone-rule takes, drops and clears, against a Python restatement
of the policies. Checks that pf_pool_fits is pf_pool_reserve's verdict, that pf_pool_zone_fits is the verdict of the
zone takes, and that slot choices, evictions and the free list follow the LRU order with ties to the lower slot."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases

HERE = os.path.dirname(os.path.abspath(__file__))
OK, NOMEM = 0, cases.capi.ERR_NOMEM


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libpool_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", os.path.join(HERE, "emu", "pool_emu.cpp"), "-o", so],
                   check=True)
    L = C.CDLL(so)
    p = C.c_void_p
    L.emu_pool_new.restype = p
    L.emu_pool_new.argtypes = [C.c_int, C.c_int, C.c_int]
    L.emu_pool_delete.argtypes = [p]
    L.emu_pool_reserve.argtypes = [p, p, C.c_int, C.c_uint32, p, p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.emu_pool_fits.argtypes = [p, p, C.c_int]
    L.emu_pool_zone_fits.argtypes = [p, p, C.c_int]
    L.emu_pool_zone_take.argtypes = [p, C.c_uint64]
    L.emu_pool_built.argtypes = [p, C.c_uint64, C.c_int]
    L.emu_pool_drop.argtypes = [p, C.c_uint64]
    L.emu_pool_reset.argtypes = [p]
    L.emu_pool_state.argtypes = [p, p, p, p, p, p, p]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Pool:
    """the policies as the parent commit's pf_pool_reserve and zone_reserve apply them"""

    def __init__(self, nkeys, mx):
        self.max = mx
        self.slot = [-1] * nkeys
        self.owner, self.has, self.touch = [-1] * mx, [0] * mx, [0] * mx
        self.free, self.used, self.nzone = [], 0, 0

    def reserve(self, keys, tick, dev):
        fresh = sorted({k for k in keys if self.slot[k] == -1})
        avail = len(self.free) + self.max - self.used
        evicted = False
        if len(fresh) > avail:
            need = len(fresh) - avail
            stamp = [max(a, int(b)) for a, b in zip(self.touch, dev)]
            pinned = {self.slot[k] for k in keys if self.slot[k] >= 0}
            cand = [s for s in range(self.used) if self.owner[s] >= 0 and s not in pinned]
            if len(cand) < need:
                return False, None, False
            cand.sort(key=lambda s: (stamp[s], s))
            for s in cand[:need]:
                self.slot[self.owner[s]] = -1
                self.has[s], self.owner[s] = 0, -1
                self.free.append(s)
            evicted = True
        for k in fresh:
            if self.free:
                s = self.free.pop()
            else:
                s, self.used = self.used, self.used + 1
            self.slot[k], self.owner[s], self.has[s] = s, k, 0
        for k in keys:
            self.touch[self.slot[k]] = tick
        return True, [self.slot[k] for k in keys], evicted

    def zone_take(self, key):
        if self.slot[key] >= 0:
            return self.slot[key]
        if self.used >= self.max:
            return -1
        self.slot[key], self.used, self.nzone = self.used, self.used + 1, self.nzone + 1
        return self.slot[key]

    def built(self, key, bits):
        if self.slot[key] >= 0:
            self.has[self.slot[key]] |= bits

    def drop(self, key):
        if self.slot[key] >= 0:
            self.has[self.slot[key]] = 0

    def reset(self):
        self.slot = [-1] * len(self.slot)
        self.owner, self.has, self.touch = [-1] * self.max, [0] * self.max, [0] * self.max
        self.free, self.used, self.nzone = [], 0, 0


def _state(L, h, nkeys, mx):
    slot, owner = np.zeros(nkeys, np.int32), np.zeros(mx, np.int64)
    has, touch, free = np.zeros(mx, np.uint8), np.zeros(mx, np.uint32), np.zeros(mx, np.int32)
    cnt = np.zeros(2, np.int64)
    nfree = L.emu_pool_state(h, _p(slot), _p(owner), _p(has), _p(touch), _p(free), _p(cnt))
    return slot.tolist(), owner.tolist(), has.tolist(), touch.tolist(), free[:nfree].tolist(), cnt.tolist()


@pytest.mark.parametrize("seed", range(12))
def test_pool_policies_match_restatement(emu, seed):
    rng = np.random.default_rng(0x9001 + seed)
    ndests, chunks = int(rng.integers(1, 5)), int(rng.integers(1, 9))
    nkeys = ndests * chunks
    mx = int(rng.integers(1, nkeys + 1))
    h = emu.emu_pool_new(ndests, chunks, mx)
    ref = Pool(nkeys, mx)
    refused = zone_refused = 0
    try:
        tick = 1
        for _ in range(1500):
            op = rng.random()
            if op < 0.55:                                   # a reservation, with device stamps the ticks may have raised
                tick += int(rng.integers(0, 3))
                keys = np.array(rng.integers(0, nkeys, int(rng.integers(0, min(nkeys, mx + 3) + 1))), np.uint64)
                dev = rng.integers(0, tick + 1, mx).astype(np.uint32)
                fits = emu.emu_pool_fits(h, _p(keys), len(keys))
                slots = np.full(len(keys), -7, np.int32)
                ev, called = C.c_int(0), C.c_int(0)
                rc = emu.emu_pool_reserve(h, _p(keys), len(keys), tick, _p(dev), _p(slots), C.byref(ev), C.byref(called))
                must_evict = len({int(k) for k in keys if ref.slot[int(k)] == -1}) > len(ref.free) + mx - ref.used
                ok, rslots, revicted = ref.reserve([int(k) for k in keys], tick, dev)
                assert (rc == OK) == ok and rc in (OK, NOMEM)
                assert bool(fits) == ok, "pf_pool_fits disagrees with pf_pool_reserve"
                assert bool(called.value) == must_evict
                if ok:
                    assert slots.tolist() == rslots and bool(ev.value) == revicted
                refused += not ok
            elif op < 0.70:                                 # a zone request: takes in order, stopping at the first refusal
                keys = [int(k) for k in rng.integers(0, nkeys, int(rng.integers(1, 5)))]
                ka = np.array(keys, np.uint64)
                fits = emu.emu_pool_zone_fits(h, _p(ka), len(keys))
                all_ok = True
                for k in keys:
                    s = emu.emu_pool_zone_take(h, k)
                    assert s == ref.zone_take(k)
                    if s < 0:
                        all_ok = False
                        break
                assert bool(fits) == all_ok, "pf_pool_zone_fits disagrees with the zone takes"
                zone_refused += not all_ok
            elif op < 0.78:                                 # fields built into a slot
                k, bits = int(rng.integers(0, nkeys)), int(rng.integers(1, 4))
                emu.emu_pool_built(h, k, bits)
                ref.built(k, bits)
            elif op < 0.85:                                 # a map change drops a key's fields
                k = int(rng.integers(0, nkeys))
                emu.emu_pool_drop(h, k)
                ref.drop(k)
            elif op < 0.87:
                emu.emu_pool_reset(h)
                ref.reset()
            slot, owner, has, touch, free, (used, nzone) = _state(emu, h, nkeys, mx)
            assert slot == ref.slot and owner == ref.owner and has == ref.has and touch == ref.touch
            assert free == ref.free and used == ref.used and nzone == ref.nzone
            # every used slot is free-listed, owned or zone-held, exactly once
            held = {s for s in slot if s >= 0 and owner[s] < 0}
            assert len(free) + sum(o >= 0 for o in owner) + nzone == used and len(held) <= nzone
    finally:
        emu.emu_pool_delete(h)
    assert refused + zone_refused > 0 or mx >= nkeys
