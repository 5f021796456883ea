"""Light path expressions at the limits of include/mcrt_abi.h, without a GPU: the tables tests/test_gpu_lpe_limits.py
renders with, their sizes, and which of their states the restated paths and photons reach.

The device keeps a path's DFA state in 8 bits and a contribution's accept mask in 32, and reads labels as symbols up
to 70. So the tables here have forward or reverse states past 127, an accept mask with every bit set, 71 symbols,
and a beauty plane on bit 31. A compiler change that shrinks one of them, or a scene change that stops the paths from
reaching its high states, fails here rather than leaving the device tests short of what they are meant to reach.

The CPU restatement (tests/lpe_ref.cpp, tests/pm_lpe_ref.cpp) writes the light group of an emitter as one character;
with 64 groups the groups must stay apart from the sky and from the vertex events, which the first tests check."""
import re

import numpy as np
import pytest

from test_aovs_cpu import load_case

SEED = 0x12345678
EVENTS = ["RD", "RS", "RG", "TS", "TG"]        # event codes 0..4 (MCRT_LPE_SYM_RD .. _TG)
EVENT_CHAR = {"a": 0, "b": 1, "c": 2, "d": 3, "e": 4}
# S_b: the vertex events whose code has bit b
S = ["[" + "".join(f"<{e}>" for k, e in enumerate(EVENTS) if k >> b & 1) + "]" for b in range(3)]
# an event of S_b p vertices before the light: the forward table remembers the last three events (states past 127 on the
# glass room's paths), the reverse one the first three of a photon (past 127 when the first is a transmission)
TAIL = [f"C.*{S[b]}.{{{p}}}L" for p in range(3) for b in range(3)] + ["C.*"]
# an event of S_b p vertices after the camera, and the sky at the first or second vertex: the forward table remembers
# the first three events. A photon-mapped camera path ends at the first delta vertex after a non-delta bounce, so it
# never reaches TAIL's forward states past 127 (they need a rough transmission then a smooth event); it reaches HEAD's
# through two smooth events (C<TS><TS><RD>)
HEAD = [f"C.{{{p}}}{S[b]}.*" for p in range(3) for b in range(3)] + ["C.{0}B.*", "C.{1}B.*", "C.*"]
ALL32 = ["C.*"] * 32
N_LABEL_GROUPS = 64
LABEL_GROUPS = [i * (N_LABEL_GROUPS - 1) // 30 for i in range(31)]      # 0, 2, ..., 63: 18, 19 and 49..53 among them
LABELS = [f"C.*L'{g}'" for g in LABEL_GROUPS] + ["C.*[" + "".join(f"L'{g}'" for g in range(N_LABEL_GROUPS)) + "]"]
# 31 expressions of Progressive's caller: its beauty plane C.* takes bit 31
P31 = (["CB", "CL", "C<RD>[LB]", "C<RD>.+[LB]", "C[<RS><RG>][LB]", "C[<RS><RG>].+[LB]", "C<T.>[LB]", "C<T.>.+[LB]"]
       + [f"C<{e}>.*" for e in EVENTS] + ["C.*B", "C.*L", "C[^S]*L", "C<RD>S+L", "C(<RS>|<TS>)+B", "C.{3,}[LB]", "C.+L"]
       + [f"C.{{{k}}}[LB]" for k in range(2, 5)] + [f"C<{e}>[LB]" for e in EVENTS[1:]]
       + ["C.*<TS>.*", "C<.S>+L", "C<RD>B", "C<TS><TS>B"])
GLASS_ROOM = "glass_room"                      # rough glass walls: photons whose first event is <TG>


def label_ids(scene):
    return np.arange(scene.n_lights, dtype=np.uint32) % N_LABEL_GROUPS


def symbol_of(mcrt, t, ch):
    """the table symbol of one character of the restatement's encoding (tests/lpe_ref.py)"""
    import lpe_ref
    if ch in EVENT_CHAR:
        return EVENT_CHAR[ch]
    if ch == "B":
        return mcrt.LPE_SYM_B
    if ch == lpe_ref.UNGROUPED:
        return mcrt.LPE_SYM_L
    return int(t["group_symbol"][ord(ch) - ord(lpe_ref.group_char(0))])


def forward_states(mcrt, t, s):
    """the forward states after each event of a string C e1 .. ek (until DEAD)"""
    out, r = [], 0
    for ch in s[1:]:
        r = int(t["next"][r, symbol_of(mcrt, t, ch)])
        if r == mcrt.LPE_DEAD:
            break
        out.append(r)
    return out


def reverse_state(mcrt, t, light_sym, events):
    """the reverse table over a photon's light, then its events in emission order"""
    r = t["rev_start"]
    for sym in [light_sym] + [EVENT_CHAR[c] for c in events]:
        if r == mcrt.LPE_DEAD:
            break
        r = int(t["rev_next"][r, sym])
    return r


_STRINGS = {}


def smooth_mesh_strings(mcrt, grouped):
    """tests/lpe_ref.cpp's strings of smooth_mesh_64 (320 lights), in N_LABEL_GROUPS groups or without groups"""
    import lpe_ref
    if grouped not in _STRINGS:
        scene, seed = load_case(mcrt, "smooth_mesh_64")
        cam = scene.cameras()[0]
        ids = label_ids(scene) if grouped else None
        _STRINGS[grouped] = lpe_ref.render_strings(scene, cam, 0, cam.height, cam.sqrtspp, seed, ids)
    return _STRINGS[grouped]


# ---------------------------------------------------------------------------------------------- the restatement's groups
def test_group_characters_collide_with_nothing():
    import lpe_ref
    chars = [lpe_ref.group_char(g) for g in range(N_LABEL_GROUPS)]
    assert len(set(chars)) == N_LABEL_GROUPS
    assert not set(chars) & (set("CB") | set(lpe_ref.VERTEX.values()) | {lpe_ref.UNGROUPED, "?"})
    assert all(re.escape(c) == c for c in chars)
    assert all(c.encode(lpe_ref.ENCODING).decode(lpe_ref.ENCODING) == c and len(c.encode(lpe_ref.ENCODING)) == 1 for c in chars)


def test_groups_only_relabel_the_emitters(mcrt):
    """smooth_mesh_64 in 64 groups of 5 lights: with each group's character read as '*', the grouped strings are the
    group-less run's strings with the same values; C.*B and C.*L are the group-less planes, and the 64 planes C.*L'g'
    partition C.*L."""
    import lpe_ref
    grouped, plain = smooth_mesh_strings(mcrt, True), smooth_mesh_strings(mcrt, False)
    ungroup = str.maketrans({lpe_ref.group_char(g): lpe_ref.UNGROUPED for g in range(N_LABEL_GROUPS)})
    mapped = [s.translate(ungroup) for s in grouped.strings]
    assert set(mapped) == set(plain.strings)
    index = {s: k for k, s in enumerate(plain.strings)}
    n_px = plain.rows * plain.width
    a = np.zeros((n_px, len(plain.strings), 3))
    np.add.at(a, (grouped.pixel, np.array([index[mapped[k]] for k in grouped.string], np.int64)), grouped.value)
    b = np.zeros_like(a)
    np.add.at(b, (plain.pixel, plain.string), plain.value)
    assert np.allclose(a, b, rtol=1e-12, atol=1e-14), np.abs(a - b).max()
    exprs = ["C.*B", "C.*L"]
    got, want = grouped.planes(exprs), plain.planes(exprs)
    assert np.allclose(got, want, rtol=1e-12, atol=1e-14) and want[0].any() and want[1].any()
    per_group = grouped.planes([f"C.*L'{g}'" for g in range(N_LABEL_GROUPS)])
    assert all(p.any() for p in per_group)
    assert np.allclose(per_group.sum(axis=0), want[1], rtol=1e-12, atol=1e-14), np.abs(per_group.sum(axis=0) - want[1]).max()


# ---------------------------------------------------------------------------------------------- the limit tables
def test_limit_table_sizes(mcrt):
    t = mcrt.lpe_compile_photon(TAIL, 0)
    assert t["next"].shape == (249, 7) and t["rev_next"].shape == (157, 7)
    t = mcrt.lpe_compile_photon(HEAD, 0)
    assert t["next"].shape == (223, 7) and t["rev_next"].shape == (180, 7)
    t = mcrt.lpe_compile_photon(ALL32, 0)
    assert len(ALL32) == mcrt.LPE_MAX_EXPRESSIONS
    assert t["next"].shape == (1, 7) and t["rev_next"].shape == (1, 7)
    assert int(t["accept"][0]) == 0xFFFFFFFF and t["join"].tolist() == [[0xFFFFFFFF]]
    t = mcrt.lpe_compile_photon(LABELS, N_LABEL_GROUPS)
    assert len(LABELS) == mcrt.LPE_MAX_EXPRESSIONS and t["next"].shape[1] == mcrt.LPE_MAX_SYMBOLS
    assert sorted(t["group_symbol"].tolist()) == list(range(mcrt.LPE_SYM_LABEL0, mcrt.LPE_MAX_SYMBOLS))
    assert len(P31) == len(set(P31)) == mcrt.LPE_MAX_EXPRESSIONS - 1
    t = mcrt.lpe_compile_photon(P31 + ["C.*"], 0)
    assert t["next"].shape[0] > 127


def test_all32_accepts_every_string_in_every_plane(mcrt):
    t = mcrt.lpe_compile(ALL32, N_LABEL_GROUPS)
    st = smooth_mesh_strings(mcrt, True)
    for s in st.strings:
        states = forward_states(mcrt, t, s)
        assert len(states) == len(s) - 1 and int(t["accept"][states[-1]]) == 0xFFFFFFFF, s


def test_p31_puts_the_beauty_plane_on_bit_31(mcrt):
    t = mcrt.lpe_compile(P31 + ["C.*"], N_LABEL_GROUPS)
    st = smooth_mesh_strings(mcrt, True)
    for s in st.strings:
        states = forward_states(mcrt, t, s)
        assert len(states) == len(s) - 1 and int(t["accept"][states[-1]]) >> 31 == 1, s


# ---------------------------------------------------------------------------------------------- states past 127, reached
TABLES = {"TAIL": TAIL, "HEAD": HEAD, "P31": P31 + ["C.*"]}
# the path tracer's cases whose paths keep a forward state past 127 between vertices (k_shade's meta2.y bits 16-23)
FORWARD_REACH = [("TAIL", GLASS_ROOM), ("HEAD", "ior_test_nobvh_64"), ("HEAD", "smooth_mesh_64"), ("P31", "c2_hexagon_room_96")]


def path_strings(mcrt, cid):
    import lpe_ref
    if cid == "smooth_mesh_64":
        return smooth_mesh_strings(mcrt, True)
    if cid not in _STRINGS:
        scene, seed = load_case(mcrt, cid)
        cam = scene.cameras()[0]
        _STRINGS[cid] = lpe_ref.render_strings(scene, cam, 0, cam.height, cam.sqrtspp, seed, label_ids(scene))
    return _STRINGS[cid]


@pytest.mark.parametrize("table,cid", FORWARD_REACH)
def test_forward_states_kept_between_vertices_pass_127(mcrt, table, cid):
    """The state after each vertex event, which the path carries to its next vertex. (TAIL's states past 127 on
    smooth_mesh_64 are only those after the light, 216 at most: the deposit reads them, no path keeps them.)"""
    t = mcrt.lpe_compile(TABLES[table], N_LABEL_GROUPS)
    reached = max(max(forward_states(mcrt, t, s[:-1]), default=0) for s in path_strings(mcrt, cid).strings)
    print(f"{table} on {cid}: forward state {reached} of {t['next'].shape[0]}")
    assert reached >= 128


def test_tail_reverse_states_pass_127_on_glass_room_photons(mcrt):
    """photons whose first event is <TG> (the rough glass walls) take TAIL's reverse states past 127"""
    import pm_lpe_ref
    scene, _ = load_case(mcrt, GLASS_ROOM)
    t = mcrt.lpe_compile_photon(TAIL, 0)
    maps, mismatched = pm_lpe_ref.photon_events(scene, 20000, 1.0, SEED)
    assert mismatched == 0
    r = np.array([reverse_state(mcrt, t, mcrt.LPE_SYM_L, ev) for _, _, evs in maps for ev in evs])
    high = (r >= 128) & (r != mcrt.LPE_DEAD)
    print(f"TAIL on {GLASS_ROOM}: {int(high.sum())} of {len(r)} photons past reverse state 127")
    assert high.any()


def test_head_query_states_pass_127_on_pm_hexagon_room(mcrt):
    """The photon mapper's queries under HEAD: every photon's history is replaced by a marker, so each photon term's
    string is its query's camera prefix C c1..ck x, then the marker"""
    import pm_lpe_ref
    from material_gen import golden_scene
    scene = golden_scene(mcrt, "pm_hexagon_room_64")
    t = mcrt.lpe_compile_photon(HEAD, 0)
    maps, _ = pm_lpe_ref.photon_events(scene, 20000, 1.0, SEED)
    marked = [(ph, ["#"] * len(ph)) for ph, _, _ in maps]
    cam = scene.cameras()[0].resized(64, 48, 1)
    st = pm_lpe_ref.render_strings(scene, cam, 0, cam.height, cam.sqrtspp, SEED, marked, 50, False)
    reached = 0
    for s in st.strings:
        if s.endswith("#"):
            q = forward_states(mcrt, t, s[:-1])
            if len(q) == len(s) - 2:
                reached = max(reached, q[-1])
    print(f"HEAD on pm_hexagon_room_64: query state {reached} of {t['next'].shape[0]}")
    assert reached >= 128 and reached != mcrt.LPE_DEAD
