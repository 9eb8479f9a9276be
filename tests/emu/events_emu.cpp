// tests/emu/events_emu.cpp -- TEST INFRASTRUCTURE. Runs the per-item rule of pfnav_agents_collect_events
// (permafrost-engine_b200/csrc/pfnav_events_kernel.cuh, unmodified) on CPU threads, each over a contiguous slice of the
// work list, and compacts the wanted items in work order, as the device's count / scan / compact passes do. The CUDA
// keywords the header uses are defined as plain C++. This is not a product path: nothing in libpfnav.so links or calls it,
// and it is built only by tests/test_agent_events_emu.py.
#include <stdint.h>
#include <stddef.h>
#include <thread>
#include <vector>
#include "../../include/pfnav.h"

#define __host__
#define __device__
#define __forceinline__ inline
#define __restrict__

#include "../../permafrost-engine_b200/csrc/pfnav_events_kernel.cuh"

// patches[n] and work[n] (the work list), agents: the population (uid order). out: room for n events. Returns the count.
extern "C" size_t emu_events(const pfnav_patch *patches, const pfnav_agent *agents, const uint32_t *work, int n, int nthreads,
                             pfnav_event *out)
{
    std::vector<uint8_t> want(n);
    std::vector<pfnav_event> ev(n);
    std::vector<std::thread> th;
    for (int t = 0; t < nthreads; t++)
        th.emplace_back([&, t]() {
            for (int i = (int)((long long)n * t / nthreads); i < (int)((long long)n * (t + 1) / nthreads); i++) {
                want[i] = pf_event_wanted(patches, agents, work, i) ? 1 : 0;
                if (want[i]) ev[i] = pf_event_make(patches, agents, work, i);
            }
        });
    for (auto &t : th) t.join();
    size_t k = 0;
    for (int i = 0; i < n; i++)
        if (want[i]) out[k++] = ev[i];
    return k;
}
