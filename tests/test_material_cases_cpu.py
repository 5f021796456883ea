"""Material rows and the BSDF branches the material tests (tests/test_gpu_materials.py) reach, without a GPU.

The golden packs hold only T = 0 or 1, no rough glass, no smooth conductor, no coated Oren-Nayar and no conductor at scene
IOR != 1. tests/material_gen.py builds such materials the way the reference's constructor would (pinned here on every
material of every pack) and puts them on golden geometry. MATERIAL_CASES is the table the GPU tests are parametrised over;
`reached` restates which branches of bsdf.cuh (bsdfLocal, buildInteraction's selectType, spawnRay, the BTDF and the two
Fresnel terms) and which k_shade feature instantiations one case takes, and EXPECTED is that list written out by hand: a
branch added without a case fails test_cases_reach_every_bsdf_branch by name."""
import glob
import os
from collections import namedtuple

import numpy as np
import pytest

from conftest import GOLDEN
from material_gen import GEOMETRY, INPUTS, inputs_of, material, material_set
from test_fast_mode_cases_cpu import MAT_ROUGH_FEATURES

# mats: a material_gen.material_set name; geometry: "lit" (ggx_64: 8 unit spheres, 3 lights), "sky" (oren_nayar_64: 8 spheres
# and a floor, no lights) or "nested" (ior_test_nobvh_64: 4 concentric spheres, no BVH); ior: scene IOR; flip: dirac_delta inverted
MatCase = namedtuple("MatCase", "mats geometry ior flip")
MatCase.__new__.__defaults__ = (1.0, False)

MATERIAL_CASES = [
    MatCase("rough_glass", "lit"), MatCase("rough_glass", "lit", 1.33),
    MatCase("smooth_coat", "lit"), MatCase("smooth_coat", "sky"),
    MatCase("smooth_lite", "lit"), MatCase("smooth_lite", "sky"), MatCase("smooth_lite", "lit", flip=True),
    MatCase("conductors", "lit"), MatCase("conductors", "lit", 1.33), MatCase("conductors", "lit", flip=True),
    MatCase("index_matched", "lit", 1.33), MatCase("tir", "lit", 1.33),
    MatCase("nested", "nested"), MatCase("nested_smooth", "nested"),
]


def mat_case_id(c):
    return f"{c.mats}-{c.geometry}-ior{c.ior:g}" + ("-flip" if c.flip else "")


EXPECTED = sorted([
    # k_shade<R, .., FEATS>: both feature sets in both precisions (the restatement runs float64, fast mode float32)
    "shade<f64,LITE>", "shade<f64,ALL>", "shade<f32,LITE>", "shade<f32,ALL>",
    # buildInteraction: selectType, n2, the rough-specular clamp of R
    "select<reflect_only>", "select<diffuse_only>", "select<three_way>", "n2<material>", "n2<external>", "rf_clamp",
    # bsdfLocal
    "bsdf<perfect_mirror>", "bsdf<conductor_smooth>", "bsdf<conductor_rough>", "bsdf<diffuse_only>",
    "bsdf<delta_reflect>", "bsdf<delta_refract>", "bsdf<diffuse_lobe,T=0>", "bsdf<diffuse_lobe,0<T<1>",
    "bsdf<mix,T=0>", "bsdf<mix,0<T<1>", "bsdf<mix,T=1>", "bsdf<half_vector,reflect>", "bsdf<half_vector,transmit>",
    "bsdf<F=1>",
    "diffuse<lambert>", "diffuse<oren_nayar>",
    # matSpecularTransmission: the transmittance applied from outside only, smooth and rough
    "btdf<smooth,outside>", "btdf<smooth,inside>", "btdf<rough,outside>", "btdf<rough,inside>",
    # ggxTransmission's flip, and its degenerate m at an index-matched interface
    "ggx_transmission<n1<n2>", "ggx_transmission<n1>n2>", "ggx_transmission<n1=n2>",
    "fresnel_conductor<n1=1>", "fresnel_conductor<n1!=1>", "fresnel_conductor<real<0>",
    # spawnRay
    "spawn<reflect>", "spawn<refract>", "spawn<refract_tir>", "spawn<diffuse>", "spawn<vndf>",
    # next-event estimation: skipped on dirac_delta materials, or through a non-opaque surface
    "nee<skipped>", "nee<evaluated>", "nee<through_surface>",
])


def outside_iors(case, rows):
    """IOR of the medium around each material's spheres: the scene's, or for the nested spheres the enclosing one's"""
    if case.geometry == "nested":
        return [case.ior] + [float(r["ior"]) for r in rows[:-1]]
    return [case.ior] * len(rows)


def material_branches(m, n_out, lights):
    """branches one material on a sphere surrounded by a medium of IOR n_out reaches"""
    out = set()
    T, ior, rough_s = float(m["transparency"]), float(m["ior"]), bool(m["rough_specular"])
    if lights:
        out.add("nee<skipped>" if m["dirac_delta"] else "nee<evaluated>")
        if not m["dirac_delta"] and not m["opaque"]:
            out.add("nee<through_surface>")
    if m["perfect_mirror"] or m["has_complex_ior"]:
        out |= {"select<reflect_only>", "spawn<reflect>", "n2<material>"}
        if m["perfect_mirror"]:
            out.add("bsdf<perfect_mirror>")
        else:
            out |= {"bsdf<conductor_rough>", "bsdf<half_vector,reflect>", "spawn<vndf>"} if rough_s else {"bsdf<conductor_smooth>"}
            out.add("fresnel_conductor<n1=1>" if n_out == 1.0 else "fresnel_conductor<n1!=1>")
            if (m["complex_ior_real"] < 0).any():
                out.add("fresnel_conductor<real<0>")
        return out
    if ior < 1.0:
        return out | {"select<diffuse_only>", "bsdf<diffuse_only>", "spawn<diffuse>", "n2<material>",
                      "diffuse<oren_nayar>" if m["rough"] else "diffuse<lambert>"}
    out |= {"select<three_way>", "n2<material>"}
    T_class = "T=0" if T == 0.0 else "T=1" if T == 1.0 else "0<T<1"
    if T < 1.0:
        out |= {"spawn<diffuse>", "diffuse<oren_nayar>" if m["rough"] else "diffuse<lambert>"}
    if ior != n_out:
        out.add("spawn<reflect>")
    if T > 0.0:
        out |= {"spawn<refract>", "n2<external>"}
        if ior != n_out:
            out |= {"spawn<refract_tir>", "bsdf<F=1>"}          # leaving the denser side at grazing angles
    if rough_s:
        out |= {"rf_clamp", "spawn<vndf>", "bsdf<half_vector,reflect>", f"bsdf<mix,{T_class}>"}
        if T > 0.0:
            out |= {"bsdf<half_vector,transmit>", "btdf<rough,outside>", "btdf<rough,inside>"}
            out |= ({"ggx_transmission<n1=n2>"} if ior == n_out else {"ggx_transmission<n1<n2>", "ggx_transmission<n1>n2>"})
    else:
        if ior != n_out:
            out.add("bsdf<delta_reflect>")
        if T > 0.0:
            out |= {"bsdf<delta_refract>", "btdf<smooth,outside>", "btdf<smooth,inside>"}
        if T < 1.0:
            out.add(f"bsdf<diffuse_lobe,{T_class}>")
    return out


def case_rows(mcrt, case):
    return [r for _, r in material_set(mcrt, case.mats)]


def features_of(rows):
    return "LITE" if not any(int(np.asarray([r[f] for r in rows]).any()) for f in MAT_ROUGH_FEATURES) else "ALL"


def reached(mcrt, case):
    rows = case_rows(mcrt, case)
    if case.flip:
        rows = [r.copy() for r in rows]
        for r in rows:
            r["dirac_delta"] = 1 - r["dirac_delta"]
    fe = features_of(rows)
    out = {f"shade<f64,{fe}>", f"shade<f32,{fe}>"}
    lights = case.geometry != "sky"
    for r, n_out in zip(rows, outside_iors(case, rows)):
        out |= material_branches(r, n_out, lights)
    return out


def test_cases_reach_every_bsdf_branch(mcrt):
    got = set()
    for c in MATERIAL_CASES:
        got |= reached(mcrt, c)
    assert sorted(got) == EXPECTED, (sorted(set(EXPECTED) - got), sorted(got - set(EXPECTED)))


def test_cases_hold_the_combinations_no_pack_has(mcrt):
    """the combinations no golden pack has, each present in at least one case"""
    rows = {c: case_rows(mcrt, c) for c in MATERIAL_CASES}
    def some(pred):
        return any(pred(c, r) for c, rs in rows.items() for r in rs)
    for sr in (1e-3, 0.05, 0.3, 1.0):
        for T in (0.4, 1.0):
            assert some(lambda c, r: r["a"][0] == sr and r["transparency"] == T and not r["has_complex_ior"]), (sr, T)
    for T in (0.0, 0.3, 0.7, 1.0):
        for rough in (False, True):
            assert some(lambda c, r: r["transparency"] == T and bool(r["rough"]) == rough and r["ior"] >= 1 and not r["rough_specular"]), (T, rough)
    for ior in (1.0, 1.33):
        assert some(lambda c, r: c.ior == ior and r["has_complex_ior"] and not r["rough_specular"] and (r["complex_ior_real"] < 0).any())
        assert some(lambda c, r: c.ior == ior and r["has_complex_ior"] and r["rough_specular"])
    assert some(lambda c, r: r["ior"] == c.ior and r["transparency"] > 0 and r["rough_specular"])
    assert some(lambda c, r: r["ior"] == c.ior and r["transparency"] > 0 and not r["rough_specular"])
    assert some(lambda c, r: c.ior == 1.33 and r["ior"] == 1.0)
    assert some(lambda c, r: c.geometry == "nested" and r["rough_specular"] and r["transparency"] > 0)
    assert some(lambda c, r: (np.asarray(r["transmittance"]) != 1.0).any() and r["transparency"] > 0)
    assert {features_of(case_rows(mcrt, c)) for c in MATERIAL_CASES} == {"LITE", "ALL"}
    assert GEOMETRY["nested"] == "ior_test_nobvh_64"


def test_case_ids_are_unique():
    ids = [mat_case_id(c) for c in MATERIAL_CASES]
    assert len(ids) == len(set(ids))


PACKS = sorted(glob.glob(os.path.join(GOLDEN, "*.mcrtpack")))


@pytest.mark.parametrize("pack", [os.path.basename(p)[:-9] for p in PACKS])
def test_material_rows_match_every_pack(pack, mcrt):
    """material(row's inputs) gives the row the reference's constructor gave, bit for bit (padding aside)"""
    mats = mcrt.Scene.from_pack(os.path.join(GOLDEN, pack + ".mcrtpack")).a["materials"]
    for i, row in enumerate(mats):
        got = material(mcrt, **inputs_of(row))
        for k in mcrt.MATERIAL_DTYPE.names:
            if k != "_pad":
                assert np.atleast_1d(got[k]).tobytes() == np.atleast_1d(row[k]).tobytes(), (pack, i, k, got[k], row[k])


def test_material_rows_pin_the_derived_constants(mcrt):
    # oren_nayar_64 pins A / B from roughness 0.25 to 16; ggx_64 a = (specular_roughness, specular_roughness)
    on = mcrt.Scene.from_pack(os.path.join(GOLDEN, "oren_nayar_64.mcrtpack")).a["materials"]
    assert sorted(set(on["roughness"][on["rough"] == 1].tolist())) == [0.25, 0.5, 1.0, 2.0, 4.0, 8.0, 16.0]
    ggx = mcrt.Scene.from_pack(os.path.join(GOLDEN, "ggx_64.mcrtpack")).a["materials"]
    r = ggx[ggx["rough_specular"] == 1]
    assert len(r) >= 6 and np.array_equal(r["a"][:, 0], r["specular_roughness"]) and np.array_equal(r["a"][:, 1], r["specular_roughness"])
    assert set(INPUTS) <= set(mcrt.MATERIAL_DTYPE.names)
    # the two rules no pack pins
    assert material(mcrt, transparency=0.3, ior=1.5)["opaque"] == 0 and material(mcrt, transparency=0.3, ior=1.5)["dirac_delta"] == 0
    smooth_metal = material(mcrt, complex_ior_real=(0.2, 0.9, 1.1), complex_ior_imag=(3.6, 2.4, 1.8))
    assert smooth_metal["dirac_delta"] == 1 and smooth_metal["opaque"] == 1
