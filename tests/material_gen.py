"""Material rows as the reference's Material constructor derives them (Material::computeProperties, material.cpp:97-111), and
scenes that put new materials on golden geometry, for the BSDF branches no golden pack reaches (tests/test_material_cases_cpu.py,
tests/test_gpu_materials.py).

`material(**inputs)` takes the fields a scene file sets, colours already linear as the packs store them, and fills in the
derived ones:
    A, B            Oren-Nayar: s2 = roughness^2, A = 1 - 0.5 s2 / (s2 + 0.33), B = 0.45 (s2 / (s2 + 0.09)); (1, 0) at roughness 0
    a               (specular_roughness, specular_roughness): isotropic GGX only
    rough           roughness > 0
    rough_specular  specular_roughness > 0
    has_complex_ior a complex IOR was given
    emissive        some emittance channel > 0
    opaque          transparency == 0. The packs have only 0 and 1; for 0 < T < 1 the surface lets light through, so it is not
                    opaque: paths inside it meet the external IOR and next-event rays may leave through it.
    dirac_delta     (has_complex_ior or perfect_mirror or transparency == 1) and not rough_specular. The reference compares
                    transparency with 1 within a tolerance (material.cpp:104, "transparency ~ 1"); the packs do not pin its
                    width, so this helper uses equality, which agrees for every value used here (0 to 0.7, and 1). The packs pin it for
                    mirrors, smooth glass, rough conductors and coated diffuse; for a smooth conductor the only lobe is the
                    pdf-1 reflection, so it is a delta; at 0 < T < 1 a diffuse lobe remains, so it is not. On the device the flag
                    only decides whether next-event estimation is skipped and where guide chains stop, so the cases that
                    depend on this choice also run with the flag flipped (`flip_dirac`).
Every material of every golden pack is reproduced bit for bit (tests/test_material_cases_cpu.py)."""
import os

import numpy as np

from conftest import GOLDEN

INPUTS = ("reflectance", "specular_reflectance", "transmittance", "emittance", "roughness", "specular_roughness", "ior",
          "transparency", "complex_ior_real", "complex_ior_imag", "perfect_mirror")
DEFAULTS = dict(reflectance=(1.0, 1.0, 1.0), specular_reflectance=(1.0, 1.0, 1.0), transmittance=(1.0, 1.0, 1.0),
                emittance=(0.0, 0.0, 0.0), roughness=0.0, specular_roughness=0.0, ior=-1.0, transparency=0.0,
                complex_ior_real=None, complex_ior_imag=None, perfect_mirror=False)


def material(mcrt, **inputs):
    """-> one mcrt.MATERIAL_DTYPE row from the input fields (INPUTS); complex_ior_real / _imag None: no complex IOR"""
    unknown = set(inputs) - set(INPUTS)
    assert not unknown, unknown
    m = dict(DEFAULTS, **inputs)
    row = np.zeros((), mcrt.MATERIAL_DTYPE)
    for k in ("reflectance", "specular_reflectance", "transmittance", "emittance"):
        row[k] = m[k]
    for k in ("roughness", "specular_roughness", "ior", "transparency"):
        row[k] = float(m[k])
    complex_ior = m["complex_ior_real"] is not None
    if complex_ior:
        row["complex_ior_real"] = m["complex_ior_real"]
        row["complex_ior_imag"] = m["complex_ior_imag"]
    s2 = float(m["roughness"]) * float(m["roughness"])
    row["A"] = 1.0 - 0.5 * s2 / (s2 + 0.33)
    row["B"] = 0.45 * (s2 / (s2 + 0.09))
    sr = float(m["specular_roughness"])
    row["a"] = (sr, sr)
    row["rough"] = float(m["roughness"]) > 0.0
    row["rough_specular"] = sr > 0.0
    row["has_complex_ior"] = complex_ior
    row["perfect_mirror"] = bool(m["perfect_mirror"])
    row["emissive"] = bool(np.any(np.asarray(m["emittance"]) > 0.0))
    row["opaque"] = float(m["transparency"]) == 0.0
    row["dirac_delta"] = (complex_ior or bool(m["perfect_mirror"]) or float(m["transparency"]) == 1.0) and not sr > 0.0
    return row


def inputs_of(row):
    """the input fields of a material row (the inverse of `material` on the inputs)"""
    out = {k: (tuple(float(x) for x in row[k]) if np.ndim(row[k]) else float(row[k])) for k in INPUTS
           if k not in ("complex_ior_real", "complex_ior_imag", "perfect_mirror")}
    out["perfect_mirror"] = bool(row["perfect_mirror"])
    if row["has_complex_ior"]:
        out["complex_ior_real"] = tuple(float(x) for x in row["complex_ior_real"])
        out["complex_ior_imag"] = tuple(float(x) for x in row["complex_ior_imag"])
    return out


# ------------------------------------------------------------------------------------------------------------- the materials
# metals_64's third material: a negative real IOR part in red
METAL_NEG = dict(complex_ior_real=(-0.13100490267476494, 0.8069658949704699, 1.103555874234062),
                 complex_ior_imag=(3.4661454927347197, 2.6008314514752406, 2.3872293467765875))
GOLD = dict(complex_ior_real=(0.18, 0.42, 1.37), complex_ior_imag=(3.42, 2.35, 1.77))
TINT = (0.55, 1.0, 0.8)      # green 1: the white-furnace tests need every green weight to be 1


def lambert(mcrt, **kw):
    return material(mcrt, reflectance=TINT, **kw)


def coated(mcrt, T, rough=0.0, ior=1.5, **kw):
    """smooth dielectric coat over Lambert (rough = 0) or Oren-Nayar, transparency T"""
    return material(mcrt, reflectance=TINT, roughness=rough, ior=ior, transparency=T, **kw)


def glass(mcrt, ior=1.5, T=1.0, sr=0.0, transmittance=TINT, **kw):
    return material(mcrt, reflectance=TINT, ior=ior, transparency=T, specular_roughness=sr, transmittance=transmittance, **kw)


def conductor(mcrt, ior, sr=0.0, spec=(0.9, 1.0, 0.95)):
    return material(mcrt, specular_reflectance=spec, specular_roughness=sr, **ior)


def mirror(mcrt, spec=(0.9, 1.0, 0.95)):
    return material(mcrt, specular_reflectance=spec, perfect_mirror=True)


def material_set(mcrt, name):
    """-> list of (label, row) of a named material set; each label names the material in per-group reports"""
    if name == "rough_glass":            # GGX transmission across alpha, at T = 1 and T = 0.4, entering and leaving the spheres
        return [(f"rough_glass_a{sr:g}_T{T:g}", glass(mcrt, sr=sr, T=T)) for T in (1.0, 0.4) for sr in (1e-3, 0.05, 0.3, 1.0)]
    if name == "smooth_coat":            # smooth coat over Lambert and Oren-Nayar at T in {0, 0.3, 0.7, 1}
        return ([(f"coat_lambert_T{T:g}", coated(mcrt, T)) for T in (0.0, 0.3, 0.7, 1.0)]
                + [(f"coat_oren_nayar_T{T:g}", coated(mcrt, T, rough=0.5)) for T in (0.0, 0.3, 0.7, 1.0)])
    if name == "smooth_lite":            # the same without Oren-Nayar: a LITE scene; transmittance != 1 seen from both sides
        return ([(f"coat_lambert_T{T:g}", coated(mcrt, T)) for T in (0.0, 0.3, 0.7, 1.0)]
                + [("lambert", lambert(mcrt)), ("glass_tinted", glass(mcrt, ior=1.7)), ("glass_tinted_T0.5", glass(mcrt, ior=1.3, T=0.5)),
                   ("coat_black", material(mcrt, reflectance=(0.0, 0.0, 0.0), ior=2.0))])
    if name == "conductors":             # smooth and rough conductors (negative real part included), a perfect mirror, GGX over
                                         # Lambert and a smooth coat over Oren-Nayar
        return [("conductor_smooth_neg", conductor(mcrt, METAL_NEG)), ("conductor_smooth_gold", conductor(mcrt, GOLD)),
                ("conductor_rough_neg", conductor(mcrt, METAL_NEG, sr=0.1)), ("conductor_rough_gold", conductor(mcrt, GOLD, sr=0.4)),
                ("mirror", mirror(mcrt)), ("ggx_coat_T0", glass(mcrt, T=0.0, sr=0.2)), ("coat_oren_nayar_T0", coated(mcrt, 0.0, rough=1.0)),
                ("conductor_rough_gold_a1", conductor(mcrt, GOLD, sr=1.0))]
    if name == "index_matched":          # material IOR = scene IOR (1.33), smooth and rough
        return [("matched_smooth", glass(mcrt, ior=1.33)), ("matched_rough", glass(mcrt, ior=1.33, sr=0.3)),
                ("matched_smooth_T0.4", glass(mcrt, ior=1.33, T=0.4)), ("matched_rough_T0.4", glass(mcrt, ior=1.33, T=0.4, sr=0.05))]
    if name == "tir":                    # IOR 1.0 spheres in a scene of IOR 1.33: total internal reflection from outside
        return [("air_smooth", glass(mcrt, ior=1.0)), ("air_rough", glass(mcrt, ior=1.0, sr=0.2)),
                ("air_coat_T0", coated(mcrt, 0.0, ior=1.0)), ("air_T0.5", glass(mcrt, ior=1.0, T=0.5))]
    if name == "nested":                 # ior_test_nobvh_64's concentric spheres: rough glass inside smooth glass
        return [("outer_smooth_1.4", glass(mcrt, ior=1.4)), ("rough_1.3", glass(mcrt, ior=1.3, sr=0.2)),
                ("smooth_1.2", glass(mcrt, ior=1.2)), ("rough_2.1", glass(mcrt, ior=2.1, sr=0.05, T=0.6))]
    if name == "nested_smooth":          # the same spheres, smooth only: the furnace's exact case
        return [("outer_smooth_1.4", glass(mcrt, ior=1.4)), ("smooth_1.3", glass(mcrt, ior=1.3)),
                ("smooth_1.2", glass(mcrt, ior=1.2)), ("smooth_2.1", glass(mcrt, ior=2.1))]
    raise KeyError(name)


# ------------------------------------------------------------------------------------------------------------- scenes
GEOMETRY = {"lit": "ggx_64", "sky": "oren_nayar_64", "nested": "ior_test_nobvh_64"}


def golden_scene(mcrt, name):
    return mcrt.Scene.from_pack(os.path.join(GOLDEN, name + ".mcrtpack"))


def with_materials(mcrt, scene, rows, scene_ior=None, lights=True, flip_dirac=False, fill=True):
    """`scene` with its non-emissive materials replaced by `rows` in turn (the geometry, and with it the BVH, unchanged).
    fill=False: only the first len(rows) of them. lights=False: the emissive materials are replaced as well and the light
    list emptied (a sky-lit scene). flip_dirac: the replaced materials' dirac_delta flag inverted."""
    a = dict(scene.a, **scene.extra)
    a["scene_ior"] = np.array([scene.ior if scene_ior is None else float(scene_ior)])
    mats = scene.a["materials"].copy()
    slots = [i for i in range(len(mats)) if lights is False or not mats[i]["emissive"]]
    if not fill:
        slots = slots[:len(rows)]
    rows = np.array(rows, mcrt.MATERIAL_DTYPE)
    if flip_dirac:
        rows["dirac_delta"] = 1 - rows["dirac_delta"]
    for j, i in enumerate(slots):
        mats[i] = rows[j % len(rows)]
    a["materials"] = mats
    if not lights:
        a["light_prim"] = np.zeros(0, scene.a["light_prim"].dtype)
        a["light_cdf"] = np.zeros(0, scene.a["light_cdf"].dtype)
    return mcrt.Scene(a)


def single_sphere(mcrt, row, scene_ior=1.0):
    """one unit sphere at the origin under the sky: no lights, no BVH (Scene::intersect scans the one primitive)"""
    base = golden_scene(mcrt, "oren_nayar_64")
    dt = {k: base.a[k].dtype for k in base.a}
    a = {k: np.zeros(0, dt[k]) for k in base.a}
    a["sphere_origin_radius"] = np.array([0.0, 0.0, 0.0, 1.0])
    a["prim_type"] = np.array([mcrt.PRIM_SPHERE], dt["prim_type"])
    a["prim_index"] = np.zeros(1, dt["prim_index"])
    a["prim_material"] = np.zeros(1, dt["prim_material"])
    a["prim_area"] = np.array([4.0 * np.pi])
    a["materials"] = np.array([row], mcrt.MATERIAL_DTYPE)
    a["scene_ior"] = np.array([float(scene_ior)])
    a["prim_original"] = np.zeros(1, base.extra["prim_original"].dtype)
    a["scene_bounds"] = np.array([-1.0, -1.0, -1.0, 1.0, 1.0, 1.0])
    for k in ("camera_f64", "camera_u32", "camera_film_u32", "camera_film_f64", "bvh_params"):
        a[k] = base.extra[k]
    return mcrt.Scene(a)
