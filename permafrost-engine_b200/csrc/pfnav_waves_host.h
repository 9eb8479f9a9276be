// pfnav_waves_host.h -- the device order of a field-request batch. No CUDA: pfnav_plan.cu launches what pack() writes,
// and tests/test_wave_pack_emu.py compiles this header with g++ to check the order.
//
// Flow requests that write the same field run in successive waves, one launch per wave. LOS requests go to the device in
// one launch whose kernel schedules them itself from their dependency order: a request must come after the parent it
// reads, so they are packed by depth (the root of a chain, or a request whose parent is kept outside the batch, has
// depth 0). Both orders are stable: within a wave or a depth, requests keep the order they were added in.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include <vector>
#include "../../include/pfnav.h"

// where pack() put a batch: enough to launch it again from the same bytes
struct pf_waves {
    int nf = 0, nl = 0;
    std::vector<int32_t> fwave_off;      // flow wave w: packed flow requests [fwave_off[w], fwave_off[w + 1])
    size_t o_fs = 0, o_lr = 0, o_ls = 0, bytes = 0;   // [flow reqs | flow dsts | LOS reqs | LOS dsts], 16-byte aligned
};

struct pf_wave_pack {
    // the batch in the order it was added: request, wave or depth, destination (pool slot or staging block)
    std::vector<pfnav_field_req> fr; std::vector<int32_t> fwave, fdst;
    std::vector<pfnav_los_req> lr; std::vector<int32_t> ldepth, ldst;
    pf_waves out;
    std::vector<int32_t> lpos;           // pack(): the packed position of the i-th LOS request added
    std::vector<int> chain;              // los_chain's scratch

    void clear() { fr.clear(); fwave.clear(); fdst.clear(); lr.clear(); ldepth.clear(); ldst.clear(); }
    void flow(const pfnav_field_req &q, int wave, int32_t dst) { fr.push_back(q); fwave.push_back(wave); fdst.push_back(dst); }
    // q.prev_index >= 0 names the parent among the LOS requests added before (in add order); a negative one is kept
    int los(const pfnav_los_req &q, int32_t dst)
    {
        ldepth.push_back(q.prev_index >= 0 ? ldepth[q.prev_index] + 1 : 0);
        lr.push_back(q); ldst.push_back(dst);
        return (int)lr.size() - 1;
    }
    // an LOS request whose parent is kept outside the batch, in pool slot or staging block `kept`
    int los_kept(pfnav_los_req q, int32_t dst, int32_t kept)
    {
        q.prev_index = -2; q._pad = kept;
        return los(q, dst);
    }
    // The LOS requests q[0, n) of one goal or path, each naming its parent within q (prev_index, or -1), those with
    // take(i): request i writes dst(i); a parent that is not taken is kept, and kept(p) is where it is read from.
    template <class Take, class Dst, class Kept>
    void los_chain(const pfnav_los_req *q, int n, Take &&take, Dst &&dst, Kept &&kept)
    {
        chain.assign(n, -1);
        for (int i = 0; i < n; i++) {
            if (!take(i)) continue;
            const int p = q[i].prev_index;
            if (p < 0 || chain[p] >= 0) {
                pfnav_los_req r = q[i];
                if (p >= 0) r.prev_index = chain[p];
                chain[i] = los(r, dst(i));
            } else {
                chain[i] = los_kept(q[i], dst(i), kept(p));
            }
        }
    }

    static size_t align16(size_t b) { return (b + 15) & ~(size_t)15; }
    // the bytes pack() writes, and where its sections start
    size_t layout()
    {
        out.nf = (int)fr.size(); out.nl = (int)lr.size();
        out.o_fs = align16(fr.size() * sizeof(pfnav_field_req));
        out.o_lr = out.o_fs + align16(fr.size() * 4);
        out.o_ls = out.o_lr + align16(lr.size() * sizeof(pfnav_los_req));
        return out.bytes = out.o_ls + align16(lr.size() * 4);
    }
    // writes layout()'s bytes to `dst`: flow requests stable by wave, LOS requests stable by depth with their in-batch
    // parents renumbered; fills out.fwave_off and lpos
    void pack(uint8_t *dst)
    {
        layout();
        const int nf = out.nf, nl = out.nl;
        std::vector<int32_t> &off = out.fwave_off;
        counting_order(fwave.data(), nf, off, fpos);
        for (int i = 0; i < nf; i++) {
            memcpy(dst + (size_t)fpos[i] * sizeof(pfnav_field_req), &fr[i], sizeof(pfnav_field_req));
            memcpy(dst + out.o_fs + (size_t)fpos[i] * 4, &fdst[i], 4);
        }
        counting_order(ldepth.data(), nl, loff, lpos);
        for (int i = 0; i < nl; i++) {
            pfnav_los_req q = lr[i];
            if (q.prev_index >= 0) q.prev_index = lpos[q.prev_index];
            memcpy(dst + out.o_lr + (size_t)lpos[i] * sizeof(pfnav_los_req), &q, sizeof(q));
            memcpy(dst + out.o_ls + (size_t)lpos[i] * 4, &ldst[i], 4);
        }
    }

private:
    std::vector<int32_t> fpos, loff;
    // stable counting sort by key: off[k] = first position of key k (off has max key + 2 entries), pos[i] = i's position
    static void counting_order(const int32_t *key, int n, std::vector<int32_t> &off, std::vector<int32_t> &pos)
    {
        int32_t maxk = 0;
        for (int i = 0; i < n; i++) maxk = key[i] > maxk ? key[i] : maxk;
        off.assign((size_t)maxk + 2, 0);
        for (int i = 0; i < n; i++) off[key[i] + 1]++;
        for (int32_t k = 0; k <= maxk; k++) off[k + 1] += off[k];
        pos.resize(n);
        for (int i = 0; i < n; i++) pos[i] = off[key[i]]++;
        for (int32_t k = maxk; k >= 0; k--) off[k + 1] = off[k];   // the increments left off[k] at the end of key k
        off[0] = 0;
    }
};
