"""The packer of a field-request batch (csrc/pfnav_waves_host.h, compiled with g++ through tests/emu/wave_pack_emu.cpp)
on random batches, against a Python restatement of the loops each batch kind used before the packer: the merge of a
goal's LOS chain into a batch (an in-batch parent renumbered, a parent left out of the batch kept as -2 with its pool
slot or staging block in _pad), the counting sorts by flow wave and LOS depth, and pfnav_los_fields_create's
re-ordering of caller requests. Checks the packed bytes of every section, the flow wave offsets, the renumbered parents
and the permutation pfnav_los_fields_create un-permutes its fields with."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases

HERE = os.path.dirname(os.path.abspath(__file__))
FIELD_REQ, LOS_REQ = cases.capi.FIELD_REQ, cases.capi.LOS_REQ
INPLACE = -3


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libwave_pack_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", os.path.join(HERE, "emu", "wave_pack_emu.cpp"), "-o", so],
                   check=True)
    L = C.CDLL(so)
    p = C.c_void_p
    L.emu_pack_new.restype = p
    L.emu_pack_delete.argtypes = [p]
    L.emu_pack_clear.argtypes = [p]
    L.emu_pack_flow.argtypes = [p, p, C.c_int, C.c_int32]
    L.emu_pack_los.argtypes = [p, p, C.c_int32]
    L.emu_pack_los_kept.argtypes = [p, p, C.c_int32, C.c_int32]
    L.emu_pack_los_chain.argtypes = [p, p, C.c_int, p, p, p, C.c_int32, p, C.POINTER(C.c_int)]
    L.emu_pack_layout.argtypes = [p, p]
    L.emu_pack.argtypes = [p, p, p, C.c_int, C.POINTER(C.c_int), p]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _a16(b):
    return (b + 15) & ~15


class Packer:
    def __init__(self, L):
        self.L, self.h = L, L.emu_pack_new()

    def close(self):
        self.L.emu_pack_delete(self.h)

    def flow(self, q, wave, dst):
        self.L.emu_pack_flow(self.h, _p(q), wave, dst)

    def los(self, q, dst):
        return self.L.emu_pack_los(self.h, _p(q), dst)

    def los_kept(self, q, dst, kept):
        return self.L.emu_pack_los_kept(self.h, _p(q), dst, kept)

    def los_chain(self, q, take, dst, kept, step):
        log = np.zeros(max(len(q), 1), np.int32)
        nk = C.c_int(0)
        self.L.emu_pack_los_chain(self.h, _p(q), len(q), _p(take.astype(np.uint8)), _p(dst.astype(np.int32)),
                                  _p(kept.astype(np.int32)), step, _p(log), C.byref(nk))
        return list(log[:nk.value])

    def pack(self):
        lay = np.zeros(6, np.uint64)
        self.L.emu_pack_layout(self.h, _p(lay))
        nf, nl, o_fs, o_lr, o_ls, nbytes = (int(v) for v in lay)
        out = np.zeros(nbytes + 1, np.uint8)         # one byte past the end: pack writes nothing there
        off = np.zeros(1024, np.int32)
        noff = C.c_int(0)
        lpos = np.zeros(max(nl, 1), np.int32)
        self.L.emu_pack(self.h, _p(out), _p(off), len(off), C.byref(noff), _p(lpos))
        assert out[nbytes] == 0 and noff.value <= len(off)
        return dict(nf=nf, nl=nl, o_fs=o_fs, o_lr=o_lr, o_ls=o_ls, bytes=out[:nbytes], off=off[:noff.value],
                    lpos=lpos[:nl])


class Batch:
    """the parent commit's batch: requests in merge order, flow waves, LOS depths and destinations"""

    def __init__(self):
        self.fr, self.fw, self.fs = [], [], []
        self.lr, self.ld, self.ls = [], [], []

    def flow(self, q, wave, dst):
        self.fr.append(q.copy()); self.fw.append(wave); self.fs.append(dst)

    def los(self, q, depth, dst):
        self.lr.append(q.copy()); self.ld.append(depth); self.ls.append(dst)
        return len(self.lr) - 1

    def chain(self, lr, take, dst, kept, step):
        """plan_batch / pf_job_launch: newpos, depth, and -2 with _pad for a parent left out"""
        n = len(lr)
        depth, newpos, calls = [0] * n, [-1] * n, []
        for i in range(n):
            if not take[i]:
                continue
            q = lr[i].copy()
            p = int(q["prev_index"])
            if p >= 0:
                if newpos[p] >= 0:
                    depth[i] = depth[p] + 1
                    q["prev_index"] = newpos[p]
                else:
                    q["prev_index"] = -2
                    q["_pad"] = int(kept[p]) + step * len(calls)
                    calls.append(p)
            newpos[i] = self.los(q, depth[i], int(dst[i]))
        return calls

    def pack(self):
        """the wave / depth counting sorts of the parent's four packers, in the 16-byte aligned layout"""
        nf, nl = len(self.fr), len(self.lr)
        maxw, maxd = max(self.fw, default=0), max(self.ld, default=0)
        fwave_off, lwave_off = [0] * (maxw + 2), [0] * (maxd + 2)
        for w in self.fw:
            fwave_off[w + 1] += 1
        for w in range(maxw + 1):
            fwave_off[w + 1] += fwave_off[w]
        for d in self.ld:
            lwave_off[d + 1] += 1
        for d in range(maxd + 1):
            lwave_off[d + 1] += lwave_off[d]
        hfr, hfs = np.zeros(nf, FIELD_REQ), np.zeros(nf, np.int32)
        cur = fwave_off[:-1]
        for i in range(nf):
            k = cur[self.fw[i]]; cur[self.fw[i]] += 1
            hfr[k], hfs[k] = self.fr[i], self.fs[i]
        hlr, hls = np.zeros(nl, LOS_REQ), np.zeros(nl, np.int32)
        cur2 = lwave_off[:-1]
        lnew = [0] * nl
        for i in range(nl):
            lnew[i] = cur2[self.ld[i]]; cur2[self.ld[i]] += 1
        for i in range(nl):
            q = self.lr[i].copy()
            if q["prev_index"] >= 0:
                q["prev_index"] = lnew[q["prev_index"]]
            hlr[lnew[i]], hls[lnew[i]] = q, self.ls[i]
        o_fs = _a16(nf * FIELD_REQ.itemsize)
        o_lr = o_fs + _a16(nf * 4)
        o_ls = o_lr + _a16(nl * LOS_REQ.itemsize)
        out = np.zeros(o_ls + _a16(nl * 4), np.uint8)
        for o, a in ((0, hfr), (o_fs, hfs), (o_lr, hlr), (o_ls, hls)):
            b = a.view(np.uint8)
            out[o:o + b.size] = b
        return dict(nf=nf, nl=nl, o_fs=o_fs, o_lr=o_lr, o_ls=o_ls, bytes=out, off=np.array(fwave_off, np.int32),
                    lpos=np.array(lnew, np.int32))


def _check(got, exp):
    for k in ("nf", "nl", "o_fs", "o_lr", "o_ls"):
        assert got[k] == exp[k], k
    assert (got["off"] == exp["off"]).all(), (got["off"], exp["off"])
    assert (got["lpos"] == exp["lpos"]).all()
    assert got["bytes"].size == exp["bytes"].size
    assert (got["bytes"] == exp["bytes"]).all()


def _rand_recs(rng, dtype, n):
    return np.frombuffer(rng.integers(0, 256, n * dtype.itemsize, dtype=np.uint8).tobytes(), dtype).copy()


def _goal_chain(rng, n):
    """a goal's LOS requests: a tree, each request's parent an earlier one (the first is the root)"""
    lr = _rand_recs(rng, LOS_REQ, n)
    for i in range(n):
        lr[i]["prev_index"] = -1 if i == 0 else int(rng.integers(0, i))
    return lr


def test_empty_batch(emu):
    P = Packer(emu)
    try:
        got = P.pack()
        assert got["bytes"].size == 0 and list(got["off"]) == [0, 0] and got["lpos"].size == 0
        _check(got, Batch().pack())
        # a cleared packer is empty again
        P.flow(_rand_recs(np.random.default_rng(0), FIELD_REQ, 1), 3, 7)
        P.pack()
        emu.emu_pack_clear(P.h)
        _check(P.pack(), Batch().pack())
    finally:
        P.close()


@pytest.mark.parametrize("seed", range(40))
def test_random_batches(emu, seed):
    """goal chains with parents left out (pool slot per parent, or the job's next staging block), flow waves from repeated
    slots, path-style LOS requests with in-batch or kept parents, in random interleavings; the same packer cleared and
    reused across batches, as the planner keeps it"""
    rng = np.random.default_rng(1000 + seed)
    P = Packer(emu)
    try:
        for _ in range(3):
            emu.emu_pack_clear(P.h)
            B = Batch()
            writes = {}
            for _ in range(int(rng.integers(0, 12))):
                op = int(rng.integers(0, 4))
                if op == 0:                 # flow requests, a wave later for every earlier write to the same slot
                    fr = _rand_recs(rng, FIELD_REQ, int(rng.integers(1, 8)))
                    for i in range(len(fr)):
                        s = int(rng.integers(0, 6))
                        w = writes.get(s, 0); writes[s] = w + 1
                        P.flow(fr[i:i + 1], w, s); B.flow(fr[i], w, s)
                elif op == 1:               # a flow request with an arbitrary wave
                    q = _rand_recs(rng, FIELD_REQ, 1)
                    w, s = int(rng.integers(0, 5)), int(rng.integers(-1, 50))
                    P.flow(q, w, s); B.flow(q[0], w, s)
                elif op == 2:               # a goal's chain, some fields held
                    n = int(rng.integers(1, 20))
                    lr = _goal_chain(rng, n)
                    take = rng.random(n) < rng.choice([0.3, 0.7, 1.0])
                    dst = rng.integers(0, 1000, n)
                    step = int(rng.integers(0, 2))
                    kept = rng.integers(0, 1000, n) if step == 0 else np.full(n, int(rng.integers(0, 100)))
                    assert P.los_chain(lr, take, dst, kept, step) == B.chain(lr, take, dst, kept, step)
                else:                       # path-style requests: in-batch parent, kept parent, or a root
                    q = _rand_recs(rng, LOS_REQ, 1)
                    dst = int(rng.integers(0, 1000))
                    kind = int(rng.integers(0, 3))
                    if kind == 0 and B.lr:
                        par = int(rng.integers(0, len(B.lr)))
                        q[0]["prev_index"] = par
                        assert P.los(q, dst) == B.los(q[0], B.ld[par] + 1, dst)
                    elif kind == 1:
                        kept = int(rng.integers(0, 1000))
                        r = q[0].copy(); r["prev_index"] = -2; r["_pad"] = kept
                        assert P.los_kept(q, dst, kept) == B.los(r, 0, dst)
                    else:
                        q[0]["prev_index"] = -1
                        assert P.los(q, dst) == B.los(q[0], 0, dst)
            _check(P.pack(), B.pack())
    finally:
        P.close()


def _los_create_parent(reqs):
    """pfnav_los_fields_create before the packer: depth waves, newidx / order, in-place parents as -2 behind n"""
    n = len(reqs)
    depth, inplace = [0] * n, []
    for i in range(n):
        q = reqs[i]
        dest = q["chunk_r"] == q["tgt_chunk_r"] and q["chunk_c"] == q["tgt_chunk_c"]
        if dest:
            pass
        elif q["prev_index"] == INPLACE:
            inplace.append(i)
        else:
            depth[i] = depth[q["prev_index"]] + 1
    maxd = max(depth, default=0)
    wave_off = [0] * (maxd + 2)
    for d in depth:
        wave_off[d + 1] += 1
    for w in range(maxd + 1):
        wave_off[w + 1] += wave_off[w]
    cursor = wave_off[:-1]
    newidx, order = [0] * n, [0] * n
    for i in range(n):
        newidx[i] = cursor[depth[i]]; cursor[depth[i]] += 1
        order[newidx[i]] = i
    srt = np.zeros(n, LOS_REQ)
    for k in range(n):
        srt[k] = reqs[order[k]]
        if srt[k]["prev_index"] >= 0:
            srt[k]["prev_index"] = newidx[srt[k]["prev_index"]]
    for j, i in enumerate(inplace):
        srt[newidx[i]]["prev_index"] = -2
        srt[newidx[i]]["_pad"] = n + j
    return srt, order


@pytest.mark.parametrize("seed", range(20))
def test_los_fields_create_order(emu, seed):
    """the packer driven as pfnav_los_fields_create drives it: the requests it uploads, and un-permuting the fields with
    lpos puts every field where the parent's `order` put it"""
    rng = np.random.default_rng(5000 + seed)
    n = int(rng.integers(0, 30))
    reqs = _rand_recs(rng, LOS_REQ, n)
    for i in range(n):
        kind = int(rng.integers(0, 3)) if i else 0
        if kind == 0:               # a destination chunk: no parent
            reqs[i]["chunk_r"], reqs[i]["chunk_c"] = reqs[i]["tgt_chunk_r"], reqs[i]["tgt_chunk_c"]
            reqs[i]["prev_index"] = -1
        else:
            reqs[i]["chunk_c"] = reqs[i]["tgt_chunk_c"] + 1
            reqs[i]["prev_index"] = INPLACE if kind == 1 else int(rng.integers(0, i))
    P = Packer(emu)
    try:
        ninplace = 0
        for i in range(n):
            q = reqs[i:i + 1]
            dest = q[0]["chunk_r"] == q[0]["tgt_chunk_r"] and q[0]["chunk_c"] == q[0]["tgt_chunk_c"]
            if not dest and q[0]["prev_index"] == INPLACE:
                P.los_kept(q, 0, n + ninplace)
                ninplace += 1
            else:
                P.los(q, 0)
        got = P.pack()
    finally:
        P.close()
    exp, order = _los_create_parent(reqs)
    assert (got["bytes"][got["o_lr"]:got["o_lr"] + n * LOS_REQ.itemsize] == exp.view(np.uint8)).all()
    fields = rng.integers(0, 256, (n, 8), dtype=np.uint8)        # a field per packed position
    parent_out, new_out = np.zeros_like(fields), np.zeros_like(fields)
    for k in range(n):
        parent_out[order[k]] = fields[k]
    for i in range(n):
        new_out[i] = fields[got["lpos"][i]]
    assert (parent_out == new_out).all()
