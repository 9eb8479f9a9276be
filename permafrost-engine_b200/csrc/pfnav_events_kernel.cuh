// pfnav_events_kernel.cuh -- the per-item rule of pfnav_agents_collect_events, kept in a header of its own so that
// tests/emu/events_emu.cpp runs the SAME source on CPU threads (it defines the CUDA keywords as plain C++).
// pfnav_events.cu includes it.
// Needs: <stdint.h>, include/pfnav.h.
#pragma once

// the patch flags that carry a decision the engine acts on (engine_todo != 0 is the other)
#define PF_EVENT_FLAGS (PFNAV_UPDATE_SET_STATE | PFNAV_UPDATE_SET_MOVING | PFNAV_UPDATE_SET_DEST)

// Whether work item wi gives an event: k_entity_apply applies its patch (the entity is not GARRISONED) and the patch
// carries SET_STATE, SET_MOVING, SET_DEST or an engine_todo. It reads the patch's flags, its engine_todo only when no
// such flag is set, and the entity's flag word only when the patch qualifies.
__host__ __device__ __forceinline__ bool pf_event_wanted(const pfnav_patch *__restrict__ patches,
                                                         const pfnav_agent *__restrict__ agents,
                                                         const uint32_t *__restrict__ work, int wi)
{
    if (!(patches[wi].flags & PF_EVENT_FLAGS) && patches[wi].engine_todo == 0) return false;
    return !(agents[work[wi]].flags & PFNAV_FLAG_GARRISONED);
}

// The event of work item wi, read before the apply: state_after and pos follow k_entity_apply's rules (SET_STATE writes
// next_state, then SET_MOVING writes it again; SET_POSITION writes next_pos x, z). Reads the patch's head (flags,
// next_state, next_attack), next_pos when SET_POSITION, engine_todo and next_dest, and the entity's state and position.
__host__ __device__ __forceinline__ pfnav_event pf_event_make(const pfnav_patch *__restrict__ patches,
                                                              const pfnav_agent *__restrict__ agents,
                                                              const uint32_t *__restrict__ work, int wi)
{
    const pfnav_patch &p = patches[wi];
    const uint32_t uid = work[wi];
    const pfnav_agent &a = agents[uid];
    pfnav_event e;
    e.uid = uid;
    e.flags = p.flags;
    e.todo = p.engine_todo;
    e.attack = p.next_attack;
    e.state_before = a.state;
    e.state_after = (e.flags & (PFNAV_UPDATE_SET_STATE | PFNAV_UPDATE_SET_MOVING)) ? (uint32_t)p.next_state : e.state_before;
    e.dest[0] = p.next_dest[0];
    e.dest[1] = p.next_dest[1];
    if (e.flags & PFNAV_UPDATE_SET_POSITION) {
        e.pos[0] = p.next_pos[0];
        e.pos[1] = p.next_pos[2];
    } else {
        e.pos[0] = a.pos[0];
        e.pos[1] = a.pos[1];
    }
    e._pad[0] = 0;
    e._pad[1] = 0;
    return e;
}
