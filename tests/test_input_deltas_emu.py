"""The host side of pfnav_agents_input_deltas (csrc/pfnav_inputs_host.h, compiled with g++ through
tests/emu/input_deltas_emu.cpp): record validation, per-uid folding in array order, the per-entity write rule the device
kernel runs (here on the CPU) against a numpy restatement, and the split of a job's batch into each member's own
records."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases
from inputs_ref import apply_np

capi = cases.capi
HERE = os.path.dirname(os.path.abspath(__file__))
D = capi.INPUT_DELTA
BITS = (capi.INPUT_TARGET_PREV, capi.INPUT_TARGET_DIR, capi.INPUT_ROT, capi.INPUT_SURROUND_FIELD, capi.INPUT_FORMATION)
EXT_BITS = capi.INPUT_TARGET_PREV | capi.INPUT_TARGET_DIR | capi.INPUT_ROT | capi.INPUT_SURROUND_FIELD


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libinput_deltas_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-D_GLIBCXX_ASSERTIONS", "-fPIC", "-shared",
                    os.path.join(HERE, "emu", "input_deltas_emu.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    p = C.c_void_p
    L.emu_input_merge.argtypes = [p, C.c_int, C.c_int, C.c_int, C.c_int, p, C.c_char_p]
    L.emu_input_job.argtypes = [p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, p, C.POINTER(C.c_int), C.c_char_p]
    L.emu_input_apply.argtypes = [p, p, p, C.c_int, C.c_int]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def merge(L, d, n, lo=0, hi=None, ext=True):
    d = np.ascontiguousarray(d, D)
    out = np.zeros(max(len(d), 1), D)
    err = C.create_string_buffer(256)
    k = L.emu_input_merge(_p(d) if len(d) else None, len(d), lo, n if hi is None else hi, int(ext), _p(out), err)
    return (None, err.value.decode()) if k < 0 else (out[:k].copy(), None)


def apply_c(L, ext, form, d, base=0):
    ext, form = ext.copy(), form.copy()
    d = np.ascontiguousarray(d, D)
    if len(d):
        L.emu_input_apply(_p(ext), _p(form), _p(d), len(d), base)
    return ext, form


def tables(rng, n):
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    ext["wait_prev"] = rng.integers(0, 9, n); ext["wait_ticks_left"] = rng.integers(0, 5, n)
    ext["surround_target_uid"] = np.where(rng.random(n) < 0.5, capi.NULL_UID, rng.integers(0, n, n))
    ext["using_surround_field"] = rng.integers(0, 2, n)
    ext["target_range"] = rng.random(n) * 30
    ext["target_prev_pos"] = rng.normal(size=(n, 2)) * 50
    ext["target_dir"] = rng.normal(size=(n, 4)); ext["rot"] = rng.normal(size=(n, 4))
    form = np.zeros(n, capi.FORMATION_IN)
    form["cell_pos"] = rng.normal(size=(n, 2)) * 50
    form["target_orientation"] = rng.normal(size=(n, 4))
    form["flags"] = rng.integers(0, 32, n)
    return ext, form


def random_deltas(rng, k, n, lo=0):
    d = np.zeros(k, D)
    d["uid"] = rng.integers(lo, lo + n, k)
    d["mask"] = rng.integers(0, 32, k)
    d["target_prev_pos"] = rng.normal(size=(k, 2)) * 40
    d["target_dir"] = rng.normal(size=(k, 4)); d["rot"] = rng.normal(size=(k, 4))
    d["using_surround_field"] = rng.integers(0, 2, k)
    d["_pad"] = rng.integers(0, 1 << 30, (k, 3))               # ignored
    f = d["formation"]
    for name in ("cell_pos", "cell_arrival_vdes", "cohesion", "align", "drag"):
        f[name] = rng.normal(size=(k, 2))
    f["target_orientation"] = rng.normal(size=(k, 4))
    f["flags"] = rng.integers(0, 32, k)
    f["_pad"] = rng.integers(0, 1 << 30, k)                     # the record is stored whole
    d["formation"] = f
    return d


def test_record_layout():
    assert D.itemsize == 128
    assert [D.fields[f][1] for f in ("uid", "mask", "target_prev_pos", "target_dir", "rot", "using_surround_field", "_pad",
                                     "formation")] == [0, 4, 8, 16, 32, 48, 52, 64]
    assert BITS == (1, 2, 4, 8, 16)


@pytest.mark.parametrize("seed", range(6))
def test_folded_batch_equals_records_in_order(emu, seed):
    """many records per uid: the folded batch (one record per uid, first-occurrence order, the union of the masks) and
    the raw records applied one by one leave both tables equal to the numpy restatement, byte for byte"""
    rng = np.random.default_rng(seed)
    n = 30
    ext, form = tables(rng, n)
    d = random_deltas(rng, 400, n)
    m, err = merge(emu, d, n)
    assert err is None
    assert list(m["uid"]) == list(dict.fromkeys(int(u) for u in d["uid"]))
    for u, k in zip(m["uid"], m["mask"]):
        assert k == np.bitwise_or.reduce(d["mask"][d["uid"] == u])
    want = apply_np(ext, form, d)
    for got in (apply_c(emu, ext, form, d), apply_c(emu, ext, form, m)):
        assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes()


@pytest.mark.parametrize("bit", list(BITS) + [0])
def test_every_bit_alone_and_mask_zero(emu, bit):
    """one bit writes exactly its field and nothing else of the 64-byte records; mask 0 writes nothing"""
    rng = np.random.default_rng(bit + 50)
    n = 8
    ext, form = tables(rng, n)
    d = random_deltas(rng, 5, n)
    d["mask"] = bit
    m, err = merge(emu, d, n)
    assert err is None and (m["mask"] == bit).all()
    e2, f2 = apply_c(emu, ext, form, m)
    assert (e2.tobytes(), f2.tobytes()) == tuple(x.tobytes() for x in apply_np(ext, form, d))
    touched = np.unique(d["uid"])
    field = {capi.INPUT_TARGET_PREV: "target_prev_pos", capi.INPUT_TARGET_DIR: "target_dir", capi.INPUT_ROT: "rot",
             capi.INPUT_SURROUND_FIELD: "using_surround_field"}.get(bit)
    for name in capi.MOVESTATE_EXT.names:
        same = (e2[name] == ext[name]).reshape(n, -1).all(axis=1)
        assert same.all() if name != field else same[np.setdiff1d(np.arange(n), touched)].all(), name
    if bit == capi.INPUT_FORMATION:
        last = {int(u): i for i, u in enumerate(d["uid"])}
        for u, i in last.items():
            assert f2[u].tobytes() == d["formation"][i].tobytes()
    else:
        assert f2.tobytes() == form.tobytes()


def test_validation(emu):
    n = 10
    def one(**kw):
        d = np.zeros(1, D)
        for k, v in kw.items():
            d[k] = v
        return d
    def withform(mask=capi.INPUT_FORMATION, **kw):
        d = one(uid=0, mask=mask)
        f = d["formation"].copy()
        for k, v in kw.items():
            f[k] = v
        d["formation"] = f
        return d
    ok = lambda d, **kw: merge(emu, d, n, **kw)[1] is None
    assert ok(np.zeros(0, D))
    assert ok(one(uid=9, mask=capi.INPUT_ROT))
    assert not ok(one(uid=10, mask=0))
    assert not ok(one(uid=3, mask=0), lo=4)                    # outside the own range
    assert not ok(one(uid=8, mask=0), hi=8)
    assert not ok(one(uid=0, mask=1 << 5)) and not ok(one(uid=0, mask=1 << 31))
    for bad in (np.nan, np.inf, -np.inf):
        assert not ok(one(uid=0, mask=capi.INPUT_TARGET_PREV, target_prev_pos=(0, bad)))
        assert not ok(one(uid=0, mask=capi.INPUT_TARGET_DIR, target_dir=(0, 0, bad, 1)))
        assert not ok(one(uid=0, mask=capi.INPUT_ROT, rot=(bad, 0, 0, 1)))
        for name, shape in (("cell_pos", 2), ("cell_arrival_vdes", 2), ("cohesion", 2), ("align", 2), ("drag", 2),
                            ("target_orientation", 4)):
            v = np.zeros(shape, np.float32); v[-1] = bad
            assert not ok(withform(**{name: v})), name
        # floats the mask does not select are not checked
        assert ok(one(uid=0, mask=capi.INPUT_TARGET_DIR, rot=(bad, 0, 0, 0), target_prev_pos=(bad, bad)))
        assert ok(withform(mask=capi.INPUT_ROT, cell_pos=(bad, 0)))
    assert ok(one(uid=0, mask=capi.INPUT_SURROUND_FIELD, using_surround_field=1))
    assert not ok(one(uid=0, mask=capi.INPUT_SURROUND_FIELD, using_surround_field=2))
    assert ok(one(uid=0, mask=capi.INPUT_ROT, using_surround_field=7))
    assert ok(withform(flags=31)) and not ok(withform(flags=32)) and not ok(withform(flags=1 << 31))
    assert ok(withform(mask=0, flags=99))
    # the four movestate_ext bits need a movestate_ext table; FORMATION does not need any table
    for bit in BITS[:4]:
        assert not ok(one(uid=0, mask=bit), ext=False)
    assert ok(withform(), ext=False) and ok(one(uid=0, mask=0), ext=False)
    # one bad record anywhere refuses the batch
    d = np.concatenate([one(uid=1, mask=capi.INPUT_ROT)] * 5 + [one(uid=1, mask=capi.INPUT_SURROUND_FIELD, using_surround_field=3)])
    assert not ok(d)


@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("seed", range(3))
def test_job_split(emu, world, seed):
    """members of unequal ranges (3 members over 100 entities: 34, 33, 33) each keep the folded records of their own
    uids, in first-occurrence order; the members' writes together equal the solo call's on the whole tables; every
    member sees the same any-formation verdict; a bad record for any uid refuses the batch on every member"""
    rng = np.random.default_rng(seed)
    n = 100
    ext, form = tables(rng, n)
    d = random_deltas(rng, 300, n)
    if seed == 2:
        d["mask"] &= EXT_BITS                               # no FORMATION anywhere
    d["uid"][:40] = rng.integers(0, 5, 40)                  # repeats on the first member
    bounds = [capi.mgpu_shard_range(n, r, world) for r in range(world)]
    assert world == 2 or len({hi - lo for lo, hi in bounds}) == 2
    solo, err = merge(emu, d, n)
    assert err is None
    want = apply_np(ext, form, d)
    got_e, got_f = ext.copy(), form.copy()
    err = C.create_string_buffer(256)
    for lo, hi in bounds:
        out = np.zeros(len(d), D)
        af = C.c_int(-1)
        k = emu.emu_input_job(_p(d), len(d), n, lo, hi, 1, _p(out), C.byref(af), err)
        assert k >= 0, err.value
        assert out[:k].tobytes() == solo[(solo["uid"] >= lo) & (solo["uid"] < hi)].tobytes()
        assert af.value == int(bool((d["mask"] & capi.INPUT_FORMATION).any()))
        e, f = apply_c(emu, got_e[lo:hi], got_f[lo:hi], out[:k], base=lo)
        got_e[lo:hi], got_f[lo:hi] = e, f
    assert got_e.tobytes() == want[0].tobytes() and got_f.tobytes() == want[1].tobytes()
    # refusals reach every member, whichever range holds the bad uid
    bad = d.copy()
    bad["mask"][-1] = capi.INPUT_SURROUND_FIELD; bad["using_surround_field"][-1] = 5
    far = d.copy(); far["uid"][7] = n
    for b in (bad, far):
        for lo, hi in bounds:
            out = np.zeros(len(d), D)
            af = C.c_int(0)
            assert emu.emu_input_job(_p(b), len(b), n, lo, hi, 1, _p(out), C.byref(af), err) == -1
