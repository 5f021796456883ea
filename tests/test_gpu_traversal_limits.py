"""The traversal structures at and past their capacities on the device (DESIGN.md §8), on the deep scenes of tests/deep_scene_gen.py
with the rays that fill them (their restated peaks are pinned by tests/test_traversal_peaks_cpu.py).

  order-free stack (40)   a ray that would overflow it is replayed in the reference's order: every answer is the reference's
  replay heap (96)        fixed: a call is refused exactly when a ray it replays needs more than 96 entries
  wide stack (48)         fixed: a ray whose restated bound (port.PortScene.wide_stack_bound) stays within 48 is answered; whether
                          the selected rays of a scene are refused is pinned per scene, and a refusal needs a bound above 48
  photon emission         from the light inside the innermost shell: the maps equal the restatement's
"""
import numpy as np
import pytest

import deep_scene_gen as deep
from oracle import port
from test_gpu_fast_mode import check_closest_hit
from test_gpu_materials import OUTLIERS, has_glass
from test_gpu_photon_mapper import check_emission

pytestmark = pytest.mark.gpu

REF_HEAP_CAPACITY, FAST_STACK, WIDE_STACK = 96, 40, 48
MCRT_ERR_UNSUPPORTED = -4          # include/mcrt_abi.h
# fast mode on each scene's selected rays (measured on one H100): True = refused, the wide stack overflows
FAST_REFUSED = {("shells", "octree"): True, ("shells", "binary_sah"): False, ("shells", "quaternary_sah"): False,
                ("grid", "quaternary_sah"): False}
F64, F32 = 0, 1
CASES = [("shells", "octree"), ("shells", "binary_sah"), ("shells", "quaternary_sah"), ("grid", "quaternary_sah")]
KINDS = {"shells": ["out", "in", "camera"], "grid": ["graze", "camera"]}


def case_id(c):
    return f"{c[0]}-{c[1]}"


@pytest.fixture(scope="module")
def held(mcrt):
    cache = {}

    def get(case):
        if case not in cache:
            kind, builder = case
            scene = deep.nested_shells(mcrt, builder) if kind == "shells" else deep.grazing_grid(mcrt, builder)
            sel = deep.select_rays(mcrt, scene, KINDS[kind], n=4000)
            cache[case] = (mcrt.PathTracer(scene, precision=F64, global_seed=0x2468ACE), scene, sel)
        return cache[case]
    yield get
    for pt, _, _ in cache.values():
        pt.close()


def assert_same_hits(mcrt, got, ref):
    assert np.array_equal(got["prim"], ref["prim"]), int((got["prim"] != ref["prim"]).sum())
    hit = ref["prim"] != mcrt.NO_PRIM
    assert np.array_equal(got["t"][hit], ref["t"][hit])
    interp = ref["interpolate"].astype(bool)
    assert np.array_equal(got["u"][interp], ref["u"][interp]) and np.array_equal(got["v"][interp], ref["v"][interp])


@pytest.mark.parametrize("exact", [0, 1])
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_closest_hit_is_the_reference_order_answer(case, exact, mcrt, held):
    """mcrt_trace_closest in parity mode on the selected rays: bit-equal to the reference-order restatement. The rays the device replays
    (all of them with exact_traversal, else those the search flags, overflowing stacks included) are refused exactly when their
    restated heap peak passes the heap's capacity: those are traced one by one."""
    pt, scene, sel = held(case)
    rays, ref = sel["rays"], sel["ref"]
    replayed = np.ones(len(rays), bool) if exact else sel["flagged"]
    refused = replayed & (sel["heap_peak"] > REF_HEAP_CAPACITY)
    pt.set_option("exact_traversal", exact)
    try:
        got = pt.intersect(rays[~refused])
        assert_same_hits(mcrt, got, ref[~refused])
        if not exact:
            assert pt.last_stats["replayed_rays"] == int(replayed[~refused].sum())
        for i in np.nonzero(refused)[0][:8]:
            with pytest.raises(mcrt.McrtError, match="overflow") as e:
                pt.intersect(rays[i:i + 1])
            assert e.value.code == MCRT_ERR_UNSUPPORTED
        over = np.nonzero(~replayed & (sel["heap_peak"] > REF_HEAP_CAPACITY))[0]
        if len(over):                                      # not replayed: the search's answer stands, whatever the heap would need
            assert_same_hits(mcrt, pt.intersect(rays[over]), ref[over])
    finally:
        pt.set_option("exact_traversal", 0)
    if case == ("shells", "octree"):
        assert refused.any()
    if case[0] == "shells" and not exact:
        assert (sel["stack_peak"][~refused] > FAST_STACK).any()     # stack overflows were answered, not refused


@pytest.mark.parametrize("dynamic_fetch", [0, 1])
@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_samples_match_restatement(case, dynamic_fetch, mcrt, held):
    """sampleRay on 4096 samples started on the selected rays (the ones the restatement can replay within the heap), with the
    order-free search's dynamic ray fetch forced either way: shadow rays towards the light at the bottom of the nest are occlusion
    queries through every shell."""
    pt, scene, sel = held(case)
    ok = sel["heap_peak"] <= REF_HEAP_CAPACITY
    base = sel["rays"][ok]
    rays = base[np.arange(4096) % len(base)]
    pixel = np.arange(4096, dtype=np.uint32); sample = (np.arange(4096) // len(base)).astype(np.uint32)
    ps = port.PortScene(scene)
    try:
        ref = ps.sample_rays(rays, pixel, sample, pt.global_seed)
    finally:
        ps.close()
    pt.set_option("dynamic_fetch", dynamic_fetch)
    try:
        got = pt.sampleRay(rays, pixel, sample)
    finally:
        pt.set_option("dynamic_fetch", -1)
    err = (np.abs(got - ref) / np.maximum(1.0, np.abs(ref))).max(axis=1)
    allowed = int(OUTLIERS * len(rays)) if has_glass(scene) else 0
    assert (err > 1e-9).sum() <= allowed, (int((err > 1e-9).sum()), float(err.max()))
    assert pt.last_stats["shadow_rays"] > 0


@pytest.mark.parametrize("case", CASES, ids=case_id)
def test_fast_mode_closest_hit(case, mcrt, held):
    """Fast mode against parity (test_gpu_fast_mode's bars). The wide stack keeps 48 entries. Rays whose restated bound stays within
    48 (the selected ones and 4000 camera rays) cannot overflow it: they are answered and checked. The selected rays as one call are
    refused or answered as pinned in FAST_REFUSED; a refusal needs a selected ray whose bound passes 48, an answer is checked."""
    pt, scene, sel = held(case)
    rays = np.concatenate([sel["rays"], deep.candidate_rays(mcrt, scene, "camera", 4000, 9)])
    ps = port.PortScene(scene)
    try:
        bound = ps.wide_stack_bound(rays, 1e-5 * deep.scene_scale(scene))    # float rounding of ray and boxes: a few 2^-24 of the scale
    finally:
        ps.close()
    safe = bound <= WIDE_STACK
    assert safe.sum() >= 1000
    check_closest_hit(mcrt, pt, scene, rays[safe], f"deep {case_id(case)} within bound")
    try:
        pt.intersect(sel["rays"], precision=F32)
        refused = False
    except mcrt.McrtError as e:
        assert e.code == MCRT_ERR_UNSUPPORTED and "overflow" in str(e)
        refused = True
    assert refused == FAST_REFUSED[case], refused
    if refused:
        assert bound[:len(sel["rays"])].max() > WIDE_STACK
    else:
        check_closest_hit(mcrt, pt, scene, sel["rays"], f"deep {case_id(case)} selected")


@pytest.mark.parametrize("builder", list(deep.BUILDERS))
def test_emission_from_the_inner_light(builder, mcrt):
    """Photon emission starts at the light inside the innermost shell: every emission ray walks out through the nest with the
    order-free search, overflowing stacks replayed. The maps equal the restatement's as in test_gpu_photon_mapper."""
    scene = deep.nested_shells(mcrt, builder)
    ep = dict(emissions=20000, caustic_factor=1.0, max_photons_per_octree_leaf=200, k_nearest_photons=50, direct_visualization=False,
              scene_bounds=scene.extra["scene_bounds"])
    pm = mcrt.PhotonMapper(scene, precision=F64, global_seed=0x13579BDF, emit=ep)
    ps = port.PortScene(scene)
    try:
        restated = ps.photon_pass(ep["emissions"], ep["caustic_factor"], ep["max_photons_per_octree_leaf"], ep["scene_bounds"], 0x13579BDF)
        assert sum(len(m["photons"]) for m in restated[:2]) > 0
        check_emission(pm, scene, restated, f"deep nest {builder}")
    finally:
        ps.close()
        pm.close()


def test_scene_of_2_24_primitives_is_refused(mcrt):
    """Scenes are accepted up to 2^24 - 1 primitives; the count is checked before any array is read."""
    import ctypes as C
    scene = deep.base_scene(mcrt)
    pt = mcrt.PathTracer(scene, precision=F64)
    try:
        d = scene.desc()
        d.n_prims = 1 << 24
        n = C.c_uint64()
        rc = mcrt.lib().mcrt_scene_upload(pt.ctx, C.byref(d), C.byref(n))
        assert rc == MCRT_ERR_UNSUPPORTED and "2^24" in mcrt.lib().mcrt_last_error(pt.ctx).decode()
    finally:
        pt.close()
