"""Light-path AOVs without a GPU: the CPU restatement (tests/light_path_ref.cpp), which tests/test_gpu_aovs.py holds each
device plane to, against the restatement of the reference's beauty frame, and which planes the golden scenes reach.

A plane's class is fixed by the interaction type the first vertex selects (makeInteraction, oracle/mcrt_oracle.cpp): a
perfect mirror or a complex-IOR conductor always reflects; a material whose n2 is below 1 (the diffuse rows, ior -1)
always scatters diffusely; anything else reflects with probability R and refracts with (1 - R) T. n2 is the material's
ior, or the external ior when the ray leaves a transparent material, so a transparent row can reflect whatever its ior."""
import os

import numpy as np
import pytest

import light_path_ref as lpr
from conftest import GOLDEN, golden_cases
from material_gen import glass, golden_scene, lambert, with_materials

PATH_CASES = [c for c in golden_cases() if not c.startswith("pm_")]
# generated: the hexagon room with rough glass walls and Lambert. Camera rays refract through a wall and reach the sky or
# a light at depth 1, and rough glass samples lights through its transmission lobe: no golden scene reaches the
# transmission_direct plane, because each of their glass objects is closed and a refracted ray always meets it again
GENERATED = ["glass_room"]
REFLECTION = (4, 5)
TRANSMISSION = (6, 7)


def generated_case(mcrt, name):
    assert name == "glass_room"
    return with_materials(mcrt, golden_scene(mcrt, "c2_hexagon_room_96"), [glass(mcrt, sr=0.2), lambert(mcrt)])


def load_case(mcrt, cid):
    """-> (scene, seed) of a golden or generated case"""
    if cid in GENERATED:
        return generated_case(mcrt, cid), 7
    scene = mcrt.Scene.from_pack(os.path.join(GOLDEN, cid + ".mcrtpack"))
    return scene, int(np.load(os.path.join(GOLDEN, cid + ".npz"))["seed"])


def lobes_reachable(scene):
    """-> (can some first vertex select IA_REFLECT, ... IA_REFRACT) from the materials the primitives use"""
    m = scene.a["materials"][np.unique(scene.a["prim_material"])]
    always_reflects = (m["perfect_mirror"] != 0) | (m["has_complex_ior"] != 0)
    transparent = m["transparency"] > 0
    specular = always_reflects | (m["ior"] >= 1.0) | transparent   # n2 >= 1 possible
    return bool(specular.any()), bool((specular & ~always_reflects & transparent).any())


_PLANES = {}


def planes_of(mcrt, cid):
    if cid not in _PLANES:
        scene, seed = load_case(mcrt, cid)
        cam = scene.cameras()[0]
        _PLANES[cid] = lpr.render_rows_aovs(scene, cam, 0, cam.height, cam.sqrtspp, seed, beauty=True)
    return _PLANES[cid]


def test_plane_names(mcrt):
    assert mcrt.AOV_NAMES == ("background", "emission", "diffuse_direct", "diffuse_indirect", "reflection_direct",
                              "reflection_indirect", "transmission_direct", "transmission_indirect")
    assert lpr.N_PLANES == len(mcrt.AOV_NAMES)
    assert "mcrt_render_accumulate_aovs_dev" in mcrt.ABI_SYMBOLS and hasattr(mcrt.lib(), "mcrt_render_accumulate_aovs_dev")


@pytest.mark.parametrize("cid", PATH_CASES + GENERATED)
def test_restated_planes_sum_to_beauty(cid, mcrt):
    planes, frame = planes_of(mcrt, cid)
    assert planes.shape == (8,) + frame.shape
    assert (planes >= 0).all()
    total = planes.sum(0)
    assert np.allclose(total, frame, rtol=1e-12, atol=0), np.abs(total - frame).max()


def test_every_plane_is_reached(mcrt):
    reached = np.zeros(8, bool)
    for cid in PATH_CASES + GENERATED:
        reached |= (planes_of(mcrt, cid)[0] != 0).reshape(8, -1).any(axis=1)
    assert reached.all(), [mcrt.AOV_NAMES[k] for k in np.nonzero(~reached)[0]]


@pytest.mark.parametrize("cid", PATH_CASES + GENERATED)
def test_unreachable_planes_are_zero(cid, mcrt):
    scene, _ = load_case(mcrt, cid)
    can_reflect, can_refract = lobes_reachable(scene)
    planes = planes_of(mcrt, cid)[0]
    # exactly zero where the materials rule the lobe out; on these scenes a lobe they allow always shows up
    assert planes[list(REFLECTION)].any() == can_reflect
    assert planes[list(TRANSMISSION)].any() == can_refract


def test_reachability_of_the_golden_scenes(mcrt):
    """The cases the structural-zero tests rest on: two scenes without a specular lobe, five without refraction."""
    no_reflect = [c for c in PATH_CASES if not lobes_reachable(load_case(mcrt, c)[0])[0]]
    no_refract = [c for c in PATH_CASES if not lobes_reachable(load_case(mcrt, c)[0])[1]]
    assert no_reflect == ["c1_hexagon_diffuse_256", "oren_nayar_64"]
    assert no_refract == ["c1_hexagon_diffuse_256", "ggx_64", "metals_64", "oren_nayar_64", "veach_mis_64"]
