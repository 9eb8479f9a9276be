// tests/emu/wave_pack_emu.cpp -- TEST INFRASTRUCTURE. A C ABI over the packer of a field-request batch
// (permafrost-engine_b200/csrc/pfnav_waves_host.h, unmodified), so that tests/test_wave_pack_emu.py can run it on random
// batches and check it against a Python restatement. This is not a product path: nothing in libpfnav.so links or calls
// it, and it is built only by tests/test_wave_pack_emu.py.
#include "../../permafrost-engine_b200/csrc/pfnav_waves_host.h"

extern "C" {

void *emu_pack_new() { return new pf_wave_pack; }
void emu_pack_delete(void *h) { delete (pf_wave_pack *)h; }
void emu_pack_clear(void *h) { ((pf_wave_pack *)h)->clear(); }

void emu_pack_flow(void *h, const pfnav_field_req *q, int wave, int32_t dst) { ((pf_wave_pack *)h)->flow(*q, wave, dst); }
int emu_pack_los(void *h, const pfnav_los_req *q, int32_t dst) { return ((pf_wave_pack *)h)->los(*q, dst); }
int emu_pack_los_kept(void *h, const pfnav_los_req *q, int32_t dst, int32_t kept)
{
    return ((pf_wave_pack *)h)->los_kept(*q, dst, kept);
}

// los_chain over q[0, n): take[i] selects, dst[i] is request i's destination, and kept(p) returns kept[p] + step * the
// number of kept calls before it (a pool slot per parent, or the job's next staging block), logging p into kept_log
void emu_pack_los_chain(void *h, const pfnav_los_req *q, int n, const uint8_t *take, const int32_t *dst, const int32_t *kept,
                        int32_t step, int32_t *kept_log, int *n_kept)
{
    *n_kept = 0;
    ((pf_wave_pack *)h)->los_chain(q, n, [&](int i) { return take[i] != 0; }, [&](int i) { return dst[i]; },
                                   [&](int p) { kept_log[*n_kept] = p; return kept[p] + step * (*n_kept)++; });
}

// layout: {nf, nl, o_fs, o_lr, o_ls, bytes}
void emu_pack_layout(void *h, uint64_t *out)
{
    pf_wave_pack &W = *(pf_wave_pack *)h;
    W.layout();
    const uint64_t v[6] = {(uint64_t)W.out.nf, (uint64_t)W.out.nl, W.out.o_fs, W.out.o_lr, W.out.o_ls, W.out.bytes};
    memcpy(out, v, sizeof(v));
}

// pack into out (layout's bytes); the wave offsets (*n_off entries, at most max_off) and the LOS positions
void emu_pack(void *h, uint8_t *out, int32_t *fwave_off, int max_off, int *n_off, int32_t *lpos)
{
    pf_wave_pack &W = *(pf_wave_pack *)h;
    W.pack(out);
    *n_off = (int)W.out.fwave_off.size();
    for (int i = 0; i < *n_off && i < max_off; i++) fwave_off[i] = W.out.fwave_off[i];
    for (size_t i = 0; i < W.lpos.size(); i++) lpos[i] = W.lpos[i];
}

}
