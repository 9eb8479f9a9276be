"""The three-step path that pfnav_agents_input_deltas replaces, restated in numpy for the tests: the records applied in
order, field by field, to copies of the whole movestate_ext and formation tables; and a builder of INPUT_DELTA records."""
import numpy as np

import cases

capi = cases.capi


def apply_np(ext, form, d, base=0):
    """-> (ext, form) after the records d, in order; ext / form None: no such table (a record that writes it fails)"""
    ext = None if ext is None else ext.copy()
    form = None if form is None else form.copy()
    for x in d:
        u, k = int(x["uid"]) - base, int(x["mask"])
        if k & capi.INPUT_TARGET_PREV: ext["target_prev_pos"][u] = x["target_prev_pos"]
        if k & capi.INPUT_TARGET_DIR: ext["target_dir"][u] = x["target_dir"]
        if k & capi.INPUT_ROT: ext["rot"][u] = x["rot"]
        if k & capi.INPUT_SURROUND_FIELD: ext["using_surround_field"][u] = x["using_surround_field"]
        if k & capi.INPUT_FORMATION: form[u] = x["formation"]
    return ext, form


def inputs(uids, **fields):
    """one INPUT_DELTA per uid; the mask follows from the fields given (target_prev, target_dir, rot, surround_field,
    formation: FORMATION_IN records or one record for all)"""
    bits = dict(target_prev=(capi.INPUT_TARGET_PREV, "target_prev_pos"), target_dir=(capi.INPUT_TARGET_DIR, "target_dir"),
                rot=(capi.INPUT_ROT, "rot"), surround_field=(capi.INPUT_SURROUND_FIELD, "using_surround_field"),
                formation=(capi.INPUT_FORMATION, "formation"))
    d = np.zeros(len(uids), capi.INPUT_DELTA)
    d["uid"] = uids
    for k, v in fields.items():
        bit, name = bits[k]
        d["mask"] |= bit
        d[name] = v
    return d


def random_inputs(rng, k, uids, ext=True):
    """k records for uids drawn from `uids` (repeats likely), random masks (without the ext bits when not ext), finite
    values, formation flags within the PFNAV_FORM_* bits"""
    d = np.zeros(k, capi.INPUT_DELTA)
    d["uid"] = rng.choice(np.asarray(uids), k)
    d["mask"] = rng.integers(0, 32, k) & (0x1F if ext else capi.INPUT_FORMATION)
    d["target_prev_pos"] = rng.normal(size=(k, 2)) * 40
    d["target_dir"] = cases.dir_quat(rng.normal(size=(k, 2))); d["rot"] = cases.dir_quat(rng.normal(size=(k, 2)))
    d["using_surround_field"] = rng.integers(0, 2, k)
    f = np.zeros(k, capi.FORMATION_IN)
    for name in ("cell_arrival_vdes", "cohesion", "align", "drag"):
        f[name] = rng.normal(size=(k, 2)) * 0.3
    f["cell_pos"] = rng.normal(size=(k, 2)) * 20
    f["target_orientation"] = cases.dir_quat(rng.normal(size=(k, 2)))
    f["flags"] = rng.integers(0, 32, k)
    d["formation"] = f
    return d
