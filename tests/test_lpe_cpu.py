"""Light path expressions without a GPU: the compiler (mcrt_lpe_compile_host) against Python's re.

Every event string C (vertex){0..4} (L'g' | B) over the five vertex events and three light groups is encoded one
character per event, each expression is translated into a Python regular expression over that encoding, and the
compiled table's accept mask must equal re.fullmatch for every string and every expression, alone and in one union."""
import itertools
import re

import numpy as np
import pytest

# one character per event: the camera, the vertex events, the sky, the lights of groups 0..2
ENC = {"C": "C", "RD": "a", "RS": "b", "RG": "c", "TS": "d", "TG": "e", "B": "B"}
N_GROUPS = 3
GROUP_CHARS = "".join(str(g) for g in range(N_GROUPS))
ALPHABET = set("CabcdeB" + GROUP_CHARS)
VERTEX = ["RD", "RS", "RG", "TS", "TG"]

EXPRESSIONS = [
    # the AOVs, the light groups and the beauty
    "CB", "CL", "C<RD>[LB]", "C<RD>.+[LB]", "C[<RS><RG>][LB]", "C[<RS><RG>].+[LB]", "C<T.>[LB]", "C<T.>.+[LB]", "C<RD>.+",
    "C.*L'0'", "C.*L'1'", "C.*L'2'", "C.*B", "C.*",
    # new ground
    "C<RD>L'0'", "C.{2}[LB]", "C.{3,}[LB]", "C[^S]*L", "C<RD>S+L", "C(<RS>|<TS>)+B",
    # every operator, shorthand, set form and label
    "C D? G* L'1'", "C (R|T){1,3} [B L'2']", "C[^<RD>L'1']*L", "C<.G>+.", "C<R.>{0,2}T?B", "C(D|S)(G|B)L?",
    "C.{4}L", "C[DG]{2,}[^B]", "C<..>*L'0'|CB", "C S* D S* L", "C(.)(.)?L'2'", "C<TD>*L", ".*L'1'", "C[^.]*B",
    "C((D|G)S)*(L'0'|L'2')",
]


def to_regex(expr):
    """The Python regular expression of an LPE over the one-character encoding (an independent restatement of the
    grammar of include/mcrt_abi.h)."""
    s = "".join(expr.split())
    i = 0

    def event():
        nonlocal i
        ch = s[i]
        i += 1
        if ch == "C":
            return {"C"}
        if ch == "B":
            return {"B"}
        if ch == ".":
            return set(ALPHABET)
        if ch in "DGSRT":
            return {"D": {"a"}, "G": {"c", "e"}, "S": {"b", "d"}, "R": {"a", "b", "c"}, "T": {"d", "e"}}[ch]
        if ch == "L":
            if i < len(s) and s[i] == "'":
                j = s.index("'", i + 1)
                g = s[i + 1:j]
                i = j + 1
                return {g}
            return set(GROUP_CHARS)
        if ch == "<":
            x, y = s[i], s[i + 1]
            assert s[i + 2] == ">"
            i += 3
            out = set()
            for ev in VERTEX:
                if x in (".", ev[0]) and y in (".", ev[1]):
                    out.add(ENC[ev])
            return out
        raise AssertionError(f"unexpected {ch!r} in {expr!r}")

    def cls(chars):
        return "(?!)" if not chars else "[" + "".join(sorted(chars)) + "]"

    out = []
    while i < len(s):
        ch = s[i]
        if ch in "()|*+?":
            out.append("(?:" if ch == "(" else ch)
            i += 1
        elif ch == "{":
            j = s.index("}", i)
            out.append(s[i:j + 1])
            i = j + 1
        elif ch == "[":
            i += 1
            neg = s[i] == "^"
            if neg:
                i += 1
            chars = set()
            while s[i] != "]":
                chars |= event()
            i += 1
            out.append(cls(ALPHABET - chars if neg else chars))
        else:
            out.append(cls(event()))
    return "".join(out)


def event_strings():
    """-> [(encoded string, [symbols after C])] of every C (vertex){0..4} (L'g' | B)"""
    out = []
    for k in range(5):
        for verts in itertools.product(VERTEX, repeat=k):
            for end in ["B"] + [f"L{g}" for g in range(N_GROUPS)]:
                enc = "C" + "".join(ENC[v] for v in verts) + (ENC["B"] if end == "B" else end[1])
                out.append((enc, list(verts) + [end]))
    return out


def symbol(mcrt, table, ev):
    if ev == "B":
        return mcrt.LPE_SYM_B
    if ev.startswith("L"):
        return int(table["group_symbol"][int(ev[1:])])
    return {"RD": mcrt.LPE_SYM_RD, "RS": mcrt.LPE_SYM_RS, "RG": mcrt.LPE_SYM_RG, "TS": mcrt.LPE_SYM_TS,
            "TG": mcrt.LPE_SYM_TG}[ev]


def accept_mask(mcrt, table, events):
    """Walks the table from state 0 (after C) as k_shade does; DEAD accepts nothing."""
    s = 0
    for ev in events:
        s = int(table["next"][s, symbol(mcrt, table, ev)])
        if s == mcrt.LPE_DEAD:
            return 0
    return int(table["accept"][s])


def check_against_re(mcrt, exprs):
    table = mcrt.lpe_compile(exprs, N_GROUPS)
    regs = [re.compile(to_regex(e)) for e in exprs]
    for enc, events in event_strings():
        want = sum(1 << i for i, r in enumerate(regs) if r.fullmatch(enc))
        got = accept_mask(mcrt, table, events)
        assert got == want, (enc, exprs, bin(got), bin(want))
    return table


@pytest.mark.parametrize("expr", EXPRESSIONS)
def test_expression_matches_re(mcrt, expr):
    check_against_re(mcrt, [expr])


# 32 expressions whose union stays within 255 states: each expression that tracks its own count of events multiplies
# the union's states, and all of EXPRESSIONS together need more (refused, test_limits)
UNION_32 = [e for e in EXPRESSIONS if e not in ("C[^<RD>L'1']*L", "C(D|S)(G|B)L?", "C.{4}L", "C[DG]{2,}[^B]",
                                                   "C<..>*L'0'|CB", "C S* D S* L", "C((D|G)S)*(L'0'|L'2')")]
UNION_32 += ["C<RD>L'1'", "C<RD>L'2'", "C<RS>B", "C<TS><TS>B"]


def test_union_of_32_matches_re(mcrt):
    assert len(UNION_32) == 32
    check_against_re(mcrt, UNION_32)


def live_states(mcrt, table):
    """States from which a nonzero accept mask is reachable through the table."""
    nxt, acc = table["next"], table["accept"]
    n = nxt.shape[0]
    live = {s for s in range(n) if acc[s]}
    changed = True
    while changed:
        changed = False
        for s in range(n):
            if s not in live and any(int(t) in live for t in nxt[s] if t != mcrt.LPE_DEAD):
                live.add(s)
                changed = True
    return live


@pytest.mark.parametrize("exprs", [UNION_32, ["C<RD>L"], ["C.{3,}[LB]"], ["C(<RS>|<TS>)+B", "CL'1'"]])
def test_dead_state_is_exactly_what_accepts_nothing(mcrt, exprs):
    table = mcrt.lpe_compile(exprs, N_GROUPS)
    nxt, acc = table["next"], table["accept"]
    assert acc[mcrt.LPE_DEAD] == 0
    # every state the table keeps can still accept something, and DEAD is the only state that cannot
    assert live_states(mcrt, table) == set(range(nxt.shape[0]))
    # states are numbered breadth-first from 0: every state is reachable from state 0
    seen, todo = {0}, [0]
    while todo:
        s = todo.pop()
        for t in nxt[s]:
            if t != mcrt.LPE_DEAD and int(t) not in seen:
                seen.add(int(t))
                todo.append(int(t))
    assert seen == set(range(nxt.shape[0]))


def test_symbols_and_labels(mcrt):
    t = mcrt.lpe_compile(["C.*L'2'", "C.*L'0'"], 4)
    assert t["next"].shape[1] == mcrt.LPE_SYM_LABEL0 + 2
    # labels take symbols in ascending group order; an unlabelled group reads the shared L
    assert list(t["group_symbol"]) == [mcrt.LPE_SYM_LABEL0, mcrt.LPE_SYM_L, mcrt.LPE_SYM_LABEL0 + 1, mcrt.LPE_SYM_L]
    t = mcrt.lpe_compile(["C<RD>L"], 0)
    assert t["next"].shape[1] == mcrt.LPE_SYM_LABEL0
    # C<RD>L: after C a diffuse vertex is the only event that can still lead to a match
    row = t["next"][0]
    assert [int(row[k]) == mcrt.LPE_DEAD for k in range(mcrt.LPE_SYM_LABEL0)] == [False, True, True, True, True, True, True]


def test_nothing_can_match(mcrt):
    t = mcrt.lpe_compile(["C[^.]L", "B"], 0)
    assert t["next"].shape[0] == 1 and (t["next"] == mcrt.LPE_DEAD).all() and not t["accept"].any()


def refused(mcrt, exprs, n_groups=N_GROUPS):
    with pytest.raises(mcrt.McrtError) as e:
        mcrt.lpe_compile(exprs, n_groups)
    return e.value.code, str(e.value)


@pytest.mark.parametrize("expr,offset", [("C<RX>L", 3), ("C(L", 3), ("C[L", 3), ("CQ", 1), ("C[]L", 2), ("", 0),
                                         ("C.{3,1}L", 6), ("CL'x'", 3), ("C <R D", 6), ("C)", 1), ("C.{2000}L", 6)])
def test_syntax_errors_name_expression_and_offset(mcrt, expr, offset):
    code, msg = refused(mcrt, ["CL", expr])
    assert code == -1   # MCRT_ERR_INVALID
    assert f"expression 1 \"{expr}\"" in msg and f"at offset {offset}" in msg


def test_limits(mcrt):
    code, msg = refused(mcrt, ["C.*"] * 33)
    assert code == -1 and "33 expressions" in msg
    mcrt.lpe_compile(["C.*"] * 32, 0)
    code, msg = refused(mcrt, ["C.*L'3'"])
    assert code == -1 and "label '3'" in msg
    code, msg = refused(mcrt, ["CL'0'"], 0)
    assert code == -1 and "no group table" in msg
    labels = "".join(f"L'{g}'" for g in range(65))
    code, msg = refused(mcrt, [f"C.*[{labels}]"], 65)
    assert code == -1 and "65 distinct labels" in msg
    mcrt.lpe_compile([f"C.*[{labels[:-5]}]"], 65)   # 64 labels
    code, msg = refused(mcrt, ["C.{300}L"])
    assert code == -4 and "255 live" in msg   # MCRT_ERR_UNSUPPORTED
    code, msg = refused(mcrt, EXPRESSIONS[:32])
    assert code == -4 and "255 live" in msg
    mcrt.lpe_compile(["C.{250}L"], 0)


@pytest.mark.parametrize("expr", ["C((.{100}){100}){100}L", "C(.{1000}){60}L", "C((D|S|G|T)?{1000}){8}L", "C(.?){1000}(.?){1000}L"])
def test_large_automata_are_refused_quickly(mcrt, expr):
    """Nested repetitions are refused by the NFA-size and subset-construction bounds before they stall the host."""
    import time
    t0 = time.perf_counter()
    code, msg = refused(mcrt, [expr])
    assert code == -4 and ("states" in msg or "steps" in msg), msg   # MCRT_ERR_UNSUPPORTED
    assert time.perf_counter() - t0 < 10.0


def test_aov_expressions_partition_every_string(mcrt):
    """The 8 AOV expressions of AOV_LPES accept every event string exactly once, in the plane aovPlane() names."""
    t = mcrt.lpe_compile(list(mcrt.AOV_LPES), N_GROUPS)
    for enc, events in event_strings():
        m = accept_mask(mcrt, t, events)
        assert m and m & (m - 1) == 0, enc
        plane = m.bit_length() - 1
        if len(events) == 1:
            want = 0 if events[0] == "B" else 1
        else:
            first = events[0]
            want = (2 if first == "RD" else (4 if first[0] == "R" else 6)) + (1 if len(events) > 2 else 0)
        assert plane == want, enc
    # "." matches any event, L and B included: "C<RD>.+" alone also takes the direct strings
    t = mcrt.lpe_compile(["C<RD>.+"], N_GROUPS)
    assert accept_mask(mcrt, t, ["RD", "B"]) == 1


# ---------------------------------------------------------------------------------------------- the CPU restatement
# tests/lpe_ref.cpp sums the restated reference's contributions per event string; tests/test_gpu_lpe.py holds device
# planes to it. Here it is held to the restatements the existing tests pin: its strings add up to oracle_render_rows'
# frame, and the eight AOV expressions give oracle_render_rows_aovs' planes (the same float64 sums in another order).
from test_aovs_cpu import GENERATED, PATH_CASES, load_case, planes_of  # noqa: E402

REF_CASES = PATH_CASES + GENERATED
_STRINGS = {}


def strings_of(mcrt, cid):
    import lpe_ref
    if cid not in _STRINGS:
        scene, seed = load_case(mcrt, cid)
        cam = scene.cameras()[0]
        ids = np.arange(scene.n_lights, dtype=np.uint32) % 2
        _STRINGS[cid] = lpe_ref.render_strings(scene, cam, 0, cam.height, cam.sqrtspp, seed, ids)
    return _STRINGS[cid]


@pytest.mark.parametrize("cid", REF_CASES)
def test_restated_strings_sum_to_beauty(mcrt, cid):
    st = strings_of(mcrt, cid)
    _, beauty = planes_of(mcrt, cid)
    assert np.allclose(st.beauty(), beauty, rtol=1e-12, atol=1e-14), np.abs(st.beauty() - beauty).max()
    assert np.allclose(st.planes(["C.*"])[0], beauty, rtol=1e-12, atol=1e-14)


@pytest.mark.parametrize("cid", REF_CASES)
def test_restated_aov_expressions_give_the_aov_planes(mcrt, cid):
    st = strings_of(mcrt, cid)
    aovs, _ = planes_of(mcrt, cid)
    got = st.planes(list(mcrt.AOV_LPES))
    assert np.allclose(got, aovs, rtol=1e-12, atol=1e-14), np.abs(got - aovs).max()


@pytest.mark.parametrize("cid,event", [("ior_test_nobvh_64", "b"), ("ior_test_nobvh_64", "d"), ("metals_64", "c"),
                                       ("ggx_64", "b"), ("ggx_64", "c"), ("glass_room", "c"), ("glass_room", "e")])
def test_restated_strings_reach_smooth_and_rough_events(mcrt, cid, event):
    """The cases tests/test_gpu_lpe.py holds to the restatement reach every vertex event between them, each smooth and
    rough lobe next to another one: <RS> and <TS> in ior_test_nobvh_64, <RG> in metals_64, <RS> and <RG> in ggx_64,
    <RG> and <TG> on the glass room's rough walls."""
    st = strings_of(mcrt, cid)
    assert any(event in s for s in st.strings), sorted(st.strings)[:20]
