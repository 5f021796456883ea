"""The photon mapper's light path expressions without a GPU: the reverse DFA and join of mcrt_lpe_compile_photon_host
against Python's re.

A photon-mapped contribution's string is a camera prefix C c1..ck x, read by the forward table up to the gather
vertex x, followed by a photon history e_m..e_1 L'g', which the reverse table reads in emission order (L'g' first).
join[forward state][reverse state] must be the accept mask of the whole string, for every split of every string."""
import itertools
import re
import time

import pytest

from test_lpe_cpu import ENC, EXPRESSIONS, N_GROUPS, UNION_32, VERTEX, refused, symbol, to_regex

PREFIXES = [list(v) for k in range(4) for v in itertools.product(VERTEX, repeat=k)]            # C (vertex){0..3}
HISTORIES = [list(v) + [f"L{g}"] for k in range(4) for v in itertools.product(VERTEX, repeat=k)
             for g in range(N_GROUPS)]                                                          # (vertex){0..3} L'g'


def encode(events):
    return "C" + "".join(ENC[e] if e in ENC else e[1] for e in events)


def forward_state(mcrt, t, events):
    s = 0
    for ev in events:
        s = int(t["next"][s, symbol(mcrt, t, ev)])
        if s == mcrt.LPE_DEAD:
            break
    return s


def reverse_state(mcrt, t, history):
    """The reverse table over a history in string order e_m..e_1 L'g', read as the emission pass does: light first."""
    r = t["rev_start"]
    for ev in reversed(history):
        if r == mcrt.LPE_DEAD:
            break
        r = int(t["rev_next"][r, symbol(mcrt, t, ev)])
    return r


def joined(mcrt, t, s, r):
    return 0 if s == mcrt.LPE_DEAD or r == mcrt.LPE_DEAD else int(t["join"][s, r])


def check_join_against_re(mcrt, exprs):
    t = mcrt.lpe_compile_photon(exprs, N_GROUPS)
    regs = [re.compile(to_regex(e)) for e in exprs]
    fwd = [forward_state(mcrt, t, u) for u in PREFIXES]
    rev = [reverse_state(mcrt, t, v) for v in HISTORIES]
    want = {}
    for u, s in zip(PREFIXES, fwd):
        for v, r in zip(HISTORIES, rev):
            enc = encode(u + v)
            if enc not in want:
                want[enc] = sum(1 << i for i, rg in enumerate(regs) if rg.fullmatch(enc))
            assert joined(mcrt, t, s, r) == want[enc], (enc, exprs)
    return t


@pytest.mark.parametrize("expr", EXPRESSIONS)
def test_join_matches_re(mcrt, expr):
    check_join_against_re(mcrt, [expr])


def test_union_of_32_join_matches_re(mcrt):
    check_join_against_re(mcrt, UNION_32)


@pytest.mark.parametrize("exprs", [UNION_32, ["C<RD>L"], ["C.*<TS>.*L"], ["C<RD><TS>+L", "C<.S>+L'1'"], ["C[^.]L"]])
def test_reverse_dead_state_is_exactly_what_accepts_nothing(mcrt, exprs):
    t = mcrt.lpe_compile_photon(exprs, N_GROUPS)
    nr = t["rev_next"].shape[0]
    # the photon histories that reach a kept state complete some camera prefix; the others reach DEAD
    if t["rev_start"] == mcrt.LPE_DEAD:
        assert not t["join"].any()
        return
    for r in range(nr):
        assert t["join"][:, r].any(), (exprs, r)
    # numbered breadth-first from the start: every kept state is reachable
    seen, todo = {t["rev_start"]}, [t["rev_start"]]
    while todo:
        r = todo.pop()
        for x in t["rev_next"][r]:
            if x != mcrt.LPE_DEAD and int(x) not in seen:
                seen.add(int(x))
                todo.append(int(x))
    assert seen == set(range(nr))


def test_nothing_can_match(mcrt):
    t = mcrt.lpe_compile_photon(["C[^.]L", "B"], 0)
    assert t["rev_start"] == mcrt.LPE_DEAD and not t["join"].any()


def test_reverse_overflow_still_serves_the_path_tracer(mcrt):
    """C.{7}<RD>.*L: the forward table counts to 8, the reversed one must remember the last 8 events (2^8 states)."""
    expr = ["C.{7}<RD>.*L"]
    t = mcrt.lpe_compile(expr, 0)
    assert t["next"].shape[0] < 20
    with pytest.raises(mcrt.McrtError) as e:
        mcrt.lpe_compile_photon(expr, 0)
    assert e.value.code == -4 and "255 live" in str(e.value)   # MCRT_ERR_UNSUPPORTED
    mcrt.lpe_compile_photon(["C.{6}<RD>.*L"], 0)
    # what the path tracer refuses the photon mapper refuses with the path tracer's reason
    code, msg = refused(mcrt, ["C.{300}L"])
    with pytest.raises(mcrt.McrtError) as e:
        mcrt.lpe_compile_photon(["C.{300}L"], N_GROUPS)
    assert e.value.code == code and "255 live" in str(e.value)


@pytest.mark.parametrize("exprs,bound", [(["C.{14}<RD>.*L"], "16384 automaton states"),
                                         (["C.{11}<RD>.*L", "C.*(.?){1000}L"], "subset-construction steps")])
def test_large_reverse_automata_are_refused_quickly(mcrt, exprs, bound):
    """Tables the forward side takes and the reverse side refuses, one per bound of the reverse construction: 2^15 subset
    states, and 2^12 states whose sets each hold the ~3000 NFA states of (.?){1000}."""
    t0 = time.perf_counter()
    mcrt.lpe_compile(exprs, 0)
    with pytest.raises(mcrt.McrtError) as e:
        mcrt.lpe_compile_photon(exprs, 0)
    assert e.value.code == -4 and "reversed" in str(e.value) and bound in str(e.value), str(e.value)
    assert time.perf_counter() - t0 < 10.0


@pytest.mark.parametrize("dv", [False, True])
def test_component_expressions_partition_every_string(mcrt, dv):
    """PM_COMPONENT_LPES(dv): every photon-mapped string, C (vertex){0..6} L'g', is accepted by exactly one of the four
    expressions, and the direct plane's expression takes none with direct visualization (no sky)."""
    exprs = list(mcrt.PM_COMPONENT_LPES(dv))
    t = check_join_against_re(mcrt, exprs)
    regs = [re.compile(to_regex(e)) for e in exprs]
    for k in range(7):
        for verts in itertools.product(VERTEX, repeat=k):
            enc = encode(list(verts) + ["L0"])
            hits = [i for i, rg in enumerate(regs) if rg.fullmatch(enc)]
            assert len(hits) == 1, (enc, hits)
            if dv:
                assert hits != [1], enc
    assert t["join"].shape[0] == t["next"].shape[0]
