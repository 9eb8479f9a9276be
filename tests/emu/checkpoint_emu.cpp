// tests/emu/checkpoint_emu.cpp -- TEST INFRASTRUCTURE. Runs the checkpoint segment rules of
// permafrost-engine_b200/csrc/pfnav_checkpoint_host.h (unmodified) on the CPU: the device's pack of a segment's rows
// (pf_ckpt_word_source, one 16-byte word per item, on CPU threads), and a restore's validation, range choice, record
// gather and the incref ops of the restored blocking rows (pf_ckpt_restore_op on CPU threads, compacted in uid order as
// the device's ordered compaction does). This is not a product path: nothing in libpfnav.so links or calls it, and it
// is built only by tests/test_checkpoint_emu.py.
#include <stdint.h>
#include <stddef.h>
#include <string.h>
#include <thread>
#include <vector>
#include "../../include/pfnav.h"

#include "../../permafrost-engine_b200/csrc/pfnav_checkpoint_host.h"

template <class F>
static void on_threads(size_t n, int nthreads, F f)
{
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; t++)
        th.emplace_back([&, t]() {
            for (size_t i = n * t / nthreads; i < n * (t + 1) / nthreads; i++) f(i);
        });
    for (auto &t : th) t.join();
}

extern "C" size_t emu_ckpt_size(uint32_t tables, size_t nflocks, size_t nrows) { return pf_ckpt_bytes(tables, nflocks, nrows); }

// One segment of [lo, hi) from whole-population tables (uid-indexed, as the device holds them; tables not in `tables`
// may be NULL) into out (room for emu_ckpt_size bytes). Returns the bytes written.
extern "C" size_t emu_ckpt_save(uint32_t tables, size_t n_total, size_t lo, size_t hi, int hz, const pfnav_flock *flocks,
                                size_t nflocks, const pfnav_agent *agents, const pfnav_movestate *ms, const pfnav_movestate_ext *ext,
                                const pfnav_formation_in *form, const pfnav_blocking *blk, int nthreads, uint8_t *out)
{
    const pf_ckpt_header h = pf_ckpt_header_make(tables, n_total, lo, hi, hz, nflocks);
    memcpy(out, &h, sizeof(h));
    if (nflocks) memcpy(out + sizeof(h), flocks, nflocks * sizeof(pfnav_flock));
    const pf_ckpt_row row = pf_ckpt_row_of(tables);
    const uint8_t *src[5] = {(const uint8_t *)agents, (const uint8_t *)ms, (const uint8_t *)ext, (const uint8_t *)form,
                             (const uint8_t *)blk};
    uint8_t *rows = out + sizeof(h) + nflocks * sizeof(pfnav_flock);
    on_threads((hi - lo) * row.words, nthreads, [&](size_t w) {
        const size_t i = w / row.words;
        const uint32_t q = (uint32_t)(w - i * row.words);
        int t;
        uint32_t k;
        pf_ckpt_word_source(row, tables, q, &t, &k);
        memcpy(rows + w * 16, src[t] + ((lo + i) * pf_ckpt_sizes[t] / 16 + k) * 16, 16);
    });
    return pf_ckpt_bytes(tables, nflocks, hi - lo);
}

// A restore on member `rank` of `world`: validation, then the records of the member's range into the out arrays (each
// with room for the range; NULL skips a table) and its incref ops in uid order (room for the range). out_info =
// {n_total, lo, hi, hz, nflocks, tables, nops}. Returns 0, or -1 with the reason in err and nothing written.
extern "C" int emu_ckpt_restore(const void *const *segs, const size_t *sizes, size_t nseg, int nlayers, int world, int rank,
                                pfnav_agent *agents, pfnav_movestate *ms, pfnav_movestate_ext *ext, pfnav_formation_in *form,
                                pfnav_blocking *blk, pfnav_blocker_op *ops, int nthreads, int64_t *out_info, char *err)
{
    pf_ckpt_set S;
    if (const char *e = pf_ckpt_check(segs, sizes, nseg, nlayers, S)) {
        strncpy(err, e, 255);
        return -1;
    }
    std::vector<size_t> b;
    pf_balanced_bounds(S.h.n_total, world, b);
    const size_t lo = b[rank], hi = b[rank + 1], n = hi - lo;
    pf_ckpt_gather(S, lo, hi, agents, ms, ext, form, blk);
    size_t nops = 0;
    if ((S.h.tables & PF_CKPT_BLK) && agents && blk) {
        std::vector<pfnav_blocker_op> staged(n);
        std::vector<uint8_t> has(n);
        on_threads(n, nthreads, [&](size_t i) { has[i] = pf_ckpt_restore_op(agents[i], blk[i], &staged[i]) ? 1 : 0; });
        for (size_t i = 0; i < n; i++)
            if (has[i]) ops[nops++] = staged[i];
    }
    const int64_t info[7] = {(int64_t)S.h.n_total, (int64_t)lo, (int64_t)hi, S.h.hz, S.h.nflocks, S.h.tables, (int64_t)nops};
    memcpy(out_info, info, sizeof(info));
    return 0;
}
