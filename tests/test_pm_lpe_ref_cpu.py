"""The CPU restatement of the photon mapper's event strings (tests/pm_lpe_ref.cpp) held to the restatements the existing
tests pin: its photons are oracle_photon_pass's bit for bit, its strings add up to oracle_pm_render_rows' sums and
the four component expressions give its component planes at 1e-12 (the same float64 terms, summed per string)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from oracle import port

SEED = 0x12345678
CASES = [  # emissions, caustic factor, k, direct_visualization, gather radius (None: k-NN)
    (2000, 10.0, 50, False, None),
    (2000, 10.0, 50, True, None),
    (2000, 10.0, 50, False, 0.15),
]


def scene_of(mcrt):
    return mcrt.Scene.from_pack(os.path.join(GOLDEN, "pm_hexagon_room_64.mcrtpack"))


def test_photons_equal_the_restated_pass(mcrt):
    import pm_lpe_ref
    scene = scene_of(mcrt)
    maps, mismatched = pm_lpe_ref.photon_events(scene, 2000, 10.0, SEED)
    assert mismatched == 0
    ps = port.PortScene(scene)
    try:
        caustic, glob, lights, _, _ = ps.photon_pass(2000, 10.0, 100, scene.extra["scene_bounds"], SEED)
    finally:
        ps.close()
    for which, ref in enumerate((caustic, glob)):
        ph, li, ev = maps[which]
        a = np.concatenate([ph.view(np.uint32), li[:, None]], axis=1)
        b = np.concatenate([np.asarray(ref["photons"], np.float32).reshape(-1, 8).view(np.uint32), lights[which][:, None]], axis=1)
        assert np.array_equal(a[np.lexsort(a.T[::-1])], b[np.lexsort(b.T[::-1])])
        # a caustic photon's last event is smooth; a global photon's is not, or it has none
        assert all(e and e[-1] in "bd" for e in ev) if which == 0 else all(not e or e[-1] in "ace" for e in ev)
    assert any(len(e) >= 2 for e in maps[1][2])


@pytest.mark.parametrize("emissions,cf,k,dv,radius", CASES)
def test_strings_sum_to_the_restated_frame_and_components(mcrt, emissions, cf, k, dv, radius):
    import pm_lpe_ref
    scene = scene_of(mcrt)
    cam = scene.cameras()[0].resized(32, 24, 2)
    maps, mismatched = pm_lpe_ref.photon_events(scene, emissions, cf, SEED)
    assert mismatched == 0
    ids = np.arange(scene.n_lights, dtype=np.uint32) % 2
    with_hist = [(ph, pm_lpe_ref.history(ev, li, ids)) for ph, li, ev in maps]
    r2 = (0.0, 0.0) if radius is None else (radius ** 2, radius ** 2)
    st = pm_lpe_ref.render_strings(scene, cam, 0, cam.height, cam.sqrtspp, SEED, with_hist, k, dv, r2, ids)
    ps = port.PortScene(scene)
    rpm = ps.photon_mapper(({"photons": maps[0][0].reshape(-1)}, {"photons": maps[1][0].reshape(-1)}, k, dv))
    try:
        if radius is not None:
            rpm.gather_radius(radius, radius)
        _, comp, _ = rpm.render_rows(cam, 0, cam.height, cam.sqrtspp, SEED)
    finally:
        rpm.close()
        ps.close()
    scale = max(1.0, float(np.abs(comp).max()))
    np.testing.assert_allclose(st.beauty(), comp.sum(axis=0), rtol=1e-12, atol=1e-14 * scale)
    got = st.planes(list(mcrt.PM_COMPONENT_LPES(dv)))
    np.testing.assert_allclose(got, comp, rtol=1e-12, atol=1e-14 * scale)
    assert comp[2].any() and comp[3].any()
    # the photon terms reach smooth and rough events on both sides of x
    assert any("b" in s or "d" in s for s in st.strings)
