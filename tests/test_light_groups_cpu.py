"""Light groups without a GPU: the grouping helper on every golden pack, the exported entry points, and the numpy
restatement of mcrt_light_groups_combine_dev that tests/test_gpu_light_groups.py holds the device kernel to bit for bit."""
import glob
import os

import numpy as np
import pytest

from conftest import GOLDEN

# groups of light_groups_by_emittance (the sky's plane comes on top)
EXPECTED_GROUPS = {
    "c1_hexagon_diffuse_256": 1, "c2_hexagon_room_96": 1, "film_hexagon_room_64": 1, "ggx_64": 2,
    "hexagon_room_octree_64": 1, "ior_test_nobvh_64": 1, "metals_64": 1, "oren_nayar_64": 0, "pm_hexagon_room_64": 1,
    "quadric_64": 0, "smooth_mesh_64": 1, "veach_mis_64": 3,
}


def test_every_pack_is_listed():
    packs = sorted(os.path.basename(p)[:-9] for p in glob.glob(os.path.join(GOLDEN, "*.mcrtpack")))
    assert packs == sorted(EXPECTED_GROUPS)


@pytest.mark.parametrize("cid", sorted(EXPECTED_GROUPS))
def test_groups_by_emittance(cid, mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    ids, emittance = mcrt.light_groups_by_emittance(scene)
    assert ids.dtype == np.uint32 and ids.shape == (scene.n_lights,)
    assert emittance.shape == (EXPECTED_GROUPS[cid], 3)
    a = scene.a
    em = a["materials"]["emittance"][a["prim_material"][a["light_prim"]]]
    if scene.n_lights:
        # numbered by first appearance
        first = [int(np.nonzero(ids == g)[0][0]) for g in range(len(emittance))]
        assert first == sorted(first) and first[0] == 0
        assert np.array_equal(emittance, em[first])
    for g in range(len(emittance)):
        assert np.allclose(em[ids == g], emittance[g], rtol=1e-12, atol=0)
    # different groups differ
    for g in range(len(emittance)):
        for h in range(g):
            assert not np.allclose(emittance[g], emittance[h], rtol=1e-12, atol=0)


def test_grouping_keeps_distinct_emittances_apart(mcrt):
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, "smooth_mesh_64.mcrtpack"))
    rows = scene.a["prim_material"][scene.a["light_prim"]]
    mats = scene.a["materials"].copy()
    mats[rows[5]]["emittance"] = mats[rows[5]]["emittance"] * (1 + 1e-9)
    a = dict(scene.a, **scene.extra)
    a["materials"] = mats
    ids, emittance = mcrt.light_groups_by_emittance(mcrt.Scene(a))
    assert len(emittance) == 2 and ids[5] == 1 and (np.delete(ids, 5) == 0).all()


def test_symbols_exported(mcrt):
    names = ("mcrt_set_light_groups", "mcrt_render_accumulate_groups_dev", "mcrt_light_groups_combine_dev")
    for name in names:
        assert name in mcrt.ABI_SYMBOLS
        assert hasattr(mcrt.lib(), name)


def test_combine_restatement(mcrt):
    rng = np.random.default_rng(3)
    planes = rng.normal(size=(4, 5, 7, 3))
    w = rng.normal(size=(4, 3))
    got = mcrt.light_groups_combine(planes, w)
    want = np.empty_like(planes[0])
    for i in np.ndindex(planes.shape[1:3]):
        for c in range(3):
            acc = planes[0][i][c] * w[0, c]
            for g in range(1, 4):
                acc = acc + planes[g][i][c] * w[g, c]
            want[i][c] = acc
    assert np.array_equal(got, want)
    # scalar weights per plane weight all three channels
    assert np.array_equal(mcrt.light_groups_combine(planes, w[:, 0]), mcrt.light_groups_combine(planes, np.repeat(w[:, :1], 3, 1)))
    # unit weights: the planes' sum in order
    assert np.array_equal(mcrt.light_groups_combine(planes, np.ones(4)), ((planes[0] + planes[1]) + planes[2]) + planes[3])
    with pytest.raises(mcrt.McrtError):
        mcrt.light_groups_combine(planes, np.ones(3))
