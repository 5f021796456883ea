"""CPU tests of the traversal structures' peaks (DESIGN.md §8). The restatement's reference-order traversal and order-free search report,
per ray, the largest number of entries their heap or stack held (port.PortScene.trace_peaks, trace_fast_peaks, trace_visible_peaks);
the device holds REF_HEAP_CAPACITY = 96 heap entries (intersect.cuh), FAST_STACK = 40 search-stack entries (bvh4.cuh) and
WIDE_STACK = 48 fast-mode stack entries (intersect.cuh). Here: the instrumented functions answer as the plain ones do, and the deep
scenes of tests/deep_scene_gen.py fill each structure past its capacity."""
import os

import numpy as np
import pytest

import deep_scene_gen as deep
from conftest import GOLDEN
from oracle import port

REF_HEAP_CAPACITY, FAST_STACK, WIDE_STACK = 96, 40, 48

# largest restated peaks of the rays select_rays keeps (seeded scenes and rays): (order-free stack, replay heap, occlusion-query stack,
# wide-stack bound)
PINNED = {
    ("shells", "octree"): (156, 112, 156, 354),
    ("shells", "binary_sah"): (70, 64, 70, 48),
    ("shells", "quaternary_sah"): (55, 64, 54, 75),
    ("grid", "quaternary_sah"): (13, 13, 8, 27),
}
KINDS = {"shells": ["out", "in", "camera"], "grid": ["graze", "camera"]}


def make(mcrt, kind, builder):
    return deep.nested_shells(mcrt, builder) if kind == "shells" else deep.grazing_grid(mcrt, builder)


@pytest.fixture(scope="module")
def selected(mcrt):
    cache = {}

    def get(kind, builder):
        if (kind, builder) not in cache:
            scene = make(mcrt, kind, builder)
            cache[kind, builder] = scene, deep.select_rays(mcrt, scene, KINDS[kind], n=4000)
        return cache[kind, builder]
    return get


def check_instrumented(mcrt, scene, rays):
    """trace_peaks answers as trace; trace_fast_peaks as trace_fast, and flags every ray whose stack peak passes FAST_STACK; the
    occlusion query in the device's visiting order (trace_visible_peaks) gives trace_visible's verdict wherever neither hands the ray
    to the replay. -> (heap peaks, stack peaks, occlusion stack peaks)"""
    ps = port.PortScene(scene)
    try:
        nodes, scale = mcrt.bvh4_host(scene), deep.scene_scale(scene)
        ref = ps.trace(rays)
        ref2, heap = ps.trace_peaks(rays)
        assert ref2.tobytes() == ref.tobytes()
        fast, flagged, _, _ = ps.trace_fast(nodes, scale, rays)
        fast2, flagged2, stack = ps.trace_fast_peaks(nodes, scale, rays)
        assert fast2.tobytes() == fast.tobytes() and np.array_equal(flagged2, flagged)
        assert flagged[stack > FAST_STACK].all()
        for f in ("prim", "t", "u", "v"):               # an answer that is not flagged is the reference's
            assert np.array_equal(fast[f][~flagged], ref[f][~flagged]), f
        hit = ref["prim"] != mcrt.NO_PRIM
        verdict, t = ps.trace_visible(nodes, scale, rays[hit], ref["prim"][hit])
        verdict2, t2, occ = ps.trace_visible_peaks(nodes, scale, rays[hit], ref["prim"][hit])
        decided = (verdict != 2) & (verdict2 != 2)
        assert np.array_equal(verdict[decided], verdict2[decided])
        assert np.array_equal(t, t2)
        assert (verdict2[occ > FAST_STACK] != 0).all()     # a full stack never answers "visible" on its own
        return heap, stack, occ
    finally:
        ps.close()


@pytest.mark.parametrize("cid", ["c2_hexagon_room_96", "hexagon_room_octree_64", "quadric_64"])
def test_instrumented_traversals_answer_as_the_plain_ones(cid, mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    rays = np.load(os.path.join(GOLDEN, cid + ".npz"))["tr_rays"]
    heap, stack, _ = check_instrumented(mcrt, scene, rays)
    assert heap.max() <= REF_HEAP_CAPACITY and stack.max() <= FAST_STACK


@pytest.mark.parametrize("kind,builder", list(PINNED))
def test_deep_scene_peaks(kind, builder, mcrt, selected):
    """The selected rays of each deep scene: the instrumented traversals agree with the plain ones, and the peaks are pinned. The
    octree nest passes every capacity: the order-free stack, the replay heap and the wide stack's bound."""
    scene, sel = selected(kind, builder)
    heap, stack, occ = check_instrumented(mcrt, scene, sel["rays"])
    assert np.array_equal(heap, sel["heap_peak"]) and np.array_equal(stack, sel["stack_peak"])
    got = (int(stack.max()), int(heap.max()), int(occ.max()), deep.wide_stack_bound(scene))
    assert got == PINNED[kind, builder], got
    if (kind, builder) == ("shells", "octree"):
        assert got[0] > FAST_STACK and got[1] > REF_HEAP_CAPACITY and got[3] > WIDE_STACK
    if kind == "shells":
        assert got[0] > FAST_STACK


def lamp_rays(scene, n=2000, seed=0):
    """n rays from the centroid of the scene's only light in seeded random directions: where photon emission starts"""
    i = scene.a["prim_index"][scene.a["light_prim"][0]]
    c = sum(scene.a[k].reshape(-1, 3)[i] for k in ("tri_v0", "tri_v1", "tri_v2")) / 3.0
    d = np.random.default_rng(seed).normal(size=(n, 3))
    return np.concatenate([np.repeat(c[None], n, axis=0), d / np.linalg.norm(d, axis=1, keepdims=True)], axis=1)


# per builder: (largest heap peak of lamp_rays, rays replayed with a heap peak above 96)
LAMP = {"octree": (115, 97), "binary_sah": (65, 0), "quaternary_sah": (60, 0)}


@pytest.mark.parametrize("builder", list(LAMP))
def test_rays_from_the_inner_light(builder, mcrt, selected):
    """Rays from the nest's light in every direction: under the octree builder the replay heap cannot take some of them, under the SAH
    builders every one fits. Photon emission leaves the light in fewer directions: on the device it is answered under every builder
    and equals the restatement (tests/test_gpu_traversal_limits.py::test_emission_from_the_inner_light)."""
    scene, _ = selected("shells", builder)
    rays = lamp_rays(scene)
    ps = port.PortScene(scene)
    try:
        _, heap = ps.trace_peaks(rays)
        _, flagged, _ = ps.trace_fast_peaks(mcrt.bvh4_host(scene), deep.scene_scale(scene), rays)
    finally:
        ps.close()
    assert (int(heap.max()), int((flagged & (heap > REF_HEAP_CAPACITY)).sum())) == LAMP[builder]


@pytest.mark.parametrize("kind,builder", list(PINNED))
def test_wide_stack_bound_per_ray(kind, builder, mcrt, selected):
    """The per-ray bound of fast mode's stack never passes the tree's bound, grows with the margin, and is 0 for a ray that misses the
    scene"""
    scene, sel = selected(kind, builder)
    ps = port.PortScene(scene)
    try:
        scale = deep.scene_scale(scene)
        tight, loose = ps.wide_stack_bound(sel["rays"], 0.0), ps.wide_stack_bound(sel["rays"], 1e-5 * scale)
        away = np.array([[0.0, 100.0 * scale, 0.0, 0.0, 1.0, 0.0]])
        assert ps.wide_stack_bound(away, 1e-5 * scale)[0] == 0
    finally:
        ps.close()
    assert (tight <= loose).all() and loose.max() <= deep.wide_stack_bound(scene)
