"""CPU: the oracle's any-hit loops (trace_closest / trace_shadow with seeds) against the float64 model of anyhitref.py -- per ray
against the replay of its draws, and in distribution against the order-free probabilities (anyhitcases.py) -- and the model's
own pieces against hand-computed rays, texref, and each other.  Rendered frames: emissive and shadow veils converge to their
float64 expectations (estcases' statistics), as on the device in test_gpu_anyhit_expectation.py."""
import numpy as np
import pytest

import anyhitcases as hc
import anyhitref as ah
import texref as tr

ORACLE_RAYS = 1 << 16
ORACLE_CASES = ["veils-4-1s", "veils-4-2s", "veils-13-1s", "veils-13-2s", "veils-29-2s", "ties", "textured", "mirrored", "mask",
                "occluded", "tinted"]


@pytest.mark.parametrize("name", ORACLE_CASES)
def test_oracle_matches_the_replay_and_the_expectation(oracle_mod, name):
    c = hc.case(name, ORACLE_RAYS)
    o = oracle_mod.Oracle()
    o.set_scene(c.scn)
    report = []
    if c.closest is not None:
        seeds = c.closest["seeds"].copy()
        hits = o.trace_closest(c.rays, seeds)
        hc.check_closest(c, hits, seeds, report)
        hc.check_closest_distribution(c, hits, seeds, report)
    seeds = c.shadow["seeds"].copy()
    T = o.trace_shadow(c.rays_s, seeds)
    hc.check_shadow(c, T, seeds, report)
    hc.check_shadow_distribution(c, T, seeds, report)
    print("\n".join(report))


# ---- the model ---------------------------------------------------------------------------------------------------------------
def _one_triangle(double_sided=0, **mat):
    from vk_gltf_renderer_b200.scene import Scene
    s = Scene()
    m = s.add_material(pbrBaseColorFactor=[1, 1, 1, mat.pop("alpha", 1.0)], pbrMetallicFactor=0.0, doubleSided=double_sided, **mat)
    p = s.add_primitive([[0, 0, 0], [1, 0, 0], [0, 1, 0]], [[0, 1, 2]], uv0=[[0, 0], [1, 0], [0, 1]],
                        colors=np.array([0xFFFFFFFF, 0x80FFFFFF, 0x40FFFFFF], np.uint32))
    s.add_node(p, m, [[2, 0, 0, 1], [0, 2, 0, 0], [0, 0, 2, 5], [0, 0, 0, 1]])    # world (1,0,5) (3,0,5) (1,2,5)
    return s


def test_crossings_of_hand_computed_rays():
    """front side: t = 4, (u, v) = (0.25, 0.25); back side culled for a single-sided closest ray, never for a shadow ray; tmin /
    tmax bound the crossing for both kinds; a ray 1e-7 from an edge is flagged; a mirroring node keeps the object-space facing"""
    M = ah.SceneModel(_one_triangle())
    rays = np.array([[1.5, 0.5, 9, 0, 0, 0, -1, 1e32], [1.5, 0.5, 1, 0, 0, 0, 1, 1e32], [1.5, 0.5, 9, 0, 0, 0, -1, 3.9],
                     [1.5, 0.5, 9, 4.1, 0, 0, -1, 1e32], [2.0, 1.0 - 1e-7, 9, 0, 0, 0, -1, 1e32]], np.float32)
    cr = M.crossings(rays, shadow=False)
    assert cr["n"].tolist() == [1, 0, 0, 0, 1]
    assert cr["t"][0, 0] == 4.0 and cr["u"][0, 0] == pytest.approx(0.25) and cr["v"][0, 0] == pytest.approx(0.25)
    assert cr["flag"].tolist() == [False, False, False, False, True]
    sh = M.crossings(rays, shadow=True)
    assert sh["n"].tolist() == [1, 1, 0, 0, 1]          # shadow rays: no culling, and tmin bounds them as well
    assert sh["t"][1, 0] == 4.0
    assert ah.SceneModel(_one_triangle(double_sided=1)).crossings(rays, shadow=False)["n"].tolist() == [1, 1, 0, 0, 1]
    s = _one_triangle()
    from vk_gltf_renderer_b200.scene import _glm
    m = np.array([[-2, 0, 0, 3], [0, 2, 0, 0], [0, 0, 2, 5], [0, 0, 0, 1]], np.float64)   # x mirrored: world (3,0,5) (1,0,5) (3,2,5)
    s.render_nodes[0]["objectToWorld"], s.render_nodes[0]["worldToObject"] = _glm(m), _glm(np.linalg.inv(m))
    cr = ah.SceneModel(s).crossings(rays[:2], shadow=False)
    assert cr["n"].tolist() == [1, 0] and cr["u"][0, 0] == pytest.approx(0.75) and cr["v"][0, 0] == pytest.approx(0.25)


def test_opacity_against_texref():
    """factor x level-0 texel alpha (magnification filter, wrap modes, no uvTransform) x interpolated vertex alpha, then the
    MASK cutoff"""
    rng = np.random.default_rng(4)
    tex = rng.integers(0, 256, (5, 7, 4), dtype=np.uint8)
    for mag, wrap in ((9729, tr.REPEAT), (9728, tr.MIRRORED_REPEAT), (9729, tr.CLAMP_TO_EDGE)):
        s = _one_triangle(double_sided=1, alpha=0.9, alphaMode=2)
        s.materials[0].pbrBaseColorTexture = s.add_texture_info(s.add_texture(tex, srgb=True, wrapS=wrap, wrapT=wrap, magFilter=mag),
                                                                 0, uv_transform=(3, 0, 0, 3, 0.5, 0.5))
        s.render_prims[0]["uv0"] = np.array([[-1.3, 0.2], [2.1, -0.7], [0.4, 3.3]], np.float32)
        M = ah.SceneModel(s)
        n = 400
        u, v = rng.random(n), rng.random(n)
        keep = u + v < 1
        u, v = u[keep], v[keep]
        p = np.array([1, 0, 5]) + np.stack([2 * u, 2 * v, np.zeros_like(u)], 1)
        rays = np.zeros((len(u), 8), np.float32)
        rays[:, 0:2], rays[:, 2], rays[:, 6], rays[:, 7] = p[:, :2], 9.0, -1.0, 1e32
        cr = M.crossings(rays, shadow=False)
        a, err, opq = M.opacity(cr)
        bary = np.stack([1 - cr["u"][:, 0] - cr["v"][:, 0], cr["u"][:, 0], cr["v"][:, 0]], 1)
        uv = bary @ s.render_prims[0]["uv0"].astype(np.float64)
        ref = tr.TexRef([tex], True, wrap, wrap, mag).sample_level(0, uv.astype(np.float32), mag == 9729)[:, 3]
        va = bary @ np.array([255, 128, 64]) / 255.0
        ok = np.isfinite(err[:, 0])
        assert ok.mean() > 0.95 and not opq.any()
        f = float(np.float32(0.9))
        assert np.allclose(a[ok, 0], f * ref[ok] * va[ok], rtol=1e-12, atol=1e-12)
        s.materials[0].alphaMode, s.materials[0].alphaCutoff = 1, 0.25
        a2, err2, _ = ah.SceneModel(s).opacity(cr)
        far = np.isfinite(err2[:, 0]) & ok
        assert np.array_equal(a2[far, 0], (f * ref[far] * va[far] >= 0.25).astype(np.float64))


def test_rand_replay_matches_the_oracle(oracle_mod):
    """draws() and steps_between() against the oracle's rand(); a seed chosen for a first draw lands exactly on it"""
    import ctypes as C
    L = oracle_mod.lib()
    seeds = np.array([0, 1, 12345, 0xFFFFFFFF, 2654435761], np.uint32)
    D = ah.draws(seeds, 40)
    for i, s0 in enumerate(seeds):
        s = C.c_uint32(int(s0))
        got = [L.oracle_rand(C.byref(s)) for _ in range(40)]
        assert np.array_equal(np.array(got, np.float64), D[i])
        assert ah.steps_between(seeds[i:i + 1], np.array([s.value], np.uint32))[0] == 40
    for k in (0, 1, 838861, (1 << 23) - 1):
        s = ah.seed_for_first_draw(k)
        assert ah.draws(np.array([s], np.uint32), 1)[0, 0] == k * ah.GRID
    assert ah.p_closest(0.0) == ah.GRID and ah.p_shadow(0.0) == 0.0
    assert ah.p_closest(0.5) == 0.5 + ah.GRID and ah.p_shadow(0.5) == 0.5 and ah.p_closest(1.0) == ah.p_shadow(1.0) == 1.0


def test_transmission_expectation_three_ways():
    """E[T] of a stack: the enumeration of accepted subsets, the DP over the number of accepted identical layers and a numpy
    Monte Carlo agree; with a thick material (Beer's law on the segment since the previous accepted crossing) the enumeration
    and the Monte Carlo agree"""
    rng = np.random.default_rng(9)
    K = 9
    p = np.full(K, 0.6)
    c = np.array([0.7, 0.55, 0.4])
    cr = dict(valid=np.ones((1, K), bool), t=np.arange(1, K + 1, dtype=np.float64)[None] * 0.1)
    a = np.full((1, K), 0.6)
    C3 = np.broadcast_to(c, (1, K, 3)).copy()
    thick = np.zeros((1, K), bool)
    absorb = np.zeros((1, K, 3))
    ET, _, _, _ = ah.shadow_expectation(cr, a, np.zeros((1, K), bool), C3, thick, absorb)
    dp = ah.identical_stack(K, ah.p_shadow(0.6), c)
    mc = ah.monte_carlo_transmission(np.full(K, ah.p_shadow(0.6)), C3[0], cr["t"][0], thick[0], absorb[0], 400000, rng)
    assert np.allclose(ET[0], dp, rtol=1e-12) and np.allclose(mc, dp, rtol=0, atol=4e-3)
    assert ET[0].max() < c.max() and dp[2] < dp[0]        # the clamp at 0.01 removes the deep products of the blue channel
    thick[0, 2:6] = True
    absorb[0, 2:6] = [0.8, 1.5, 3.0]
    a[0, 2:6] = [0.5, 0.3, 0.9, 0.7]
    ET2, _, _, _ = ah.shadow_expectation(cr, a, np.zeros((1, K), bool), C3, thick, absorb)
    mc2 = ah.monte_carlo_transmission(ah.p_shadow(a[0]), C3[0], cr["t"][0], thick[0], absorb[0], 400000, rng)
    assert np.allclose(mc2, ET2[0], rtol=0, atol=4e-3) and not np.allclose(ET2[0], ET[0], atol=1e-3)


# ---- the frame path ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [1, 5])
def test_oracle_emissive_veils(oracle_mod, n):
    """black BLEND layers with distinct emission in front of a constant environment: every pixel converges to
    sum_i e_i p_i prod_{j<i} (1 - p_j) + L prod_j (1 - p_j), p on the closest-hit grid"""
    import estcases as C
    from test_estimator_expectation import _render
    scn, E = hc.emissive_veils(n, C.FURNACE_L)
    w = h = 64
    acc, _, _ = _render(oracle_mod, scn, C.furnace_env(), C.frame_info(scn, w, h, {}), w, h, 48, max_depth=2)
    report = []
    ok_val, ok_sens = C.check_face(acc, np.ones((h, w), bool), E, f"emissive veils n={n}", report)
    print(report[0])
    assert ok_val and ok_sens, report[0]


def test_oracle_shadow_veils(oracle_mod):
    """the light-only faces of the furnace polyhedron behind five black BLEND layers (one of alpha 0, two single-sided facing
    away from the body): each face converges to its light-only expectation times prod_i (1 - p_i), p on the shadow grid"""
    import estcases as C
    import estref
    from test_estimator_expectation import _render
    scn, normals, case, factor = hc.shadow_veils(5)
    assert hc.veils_off_view(scn, 20) > 1.0 and 0.7 < factor < 0.85
    w = h = 256
    frames = 250
    acc, ids, o = _render(oracle_mod, scn, C.furnace_env(), C.frame_info(scn, w, h, case), w, h, frames)
    env = estref.Env.from_oracle(o)
    faces = C.face_masks(ids, 1200)
    assert len(faces) >= 4 and sum(C.expected_face(case, env, scn, normals, k, m, w, h).max() > 0 for k, m in faces.items()) >= 2
    report, bad = [], []
    for k, m in faces.items():
        E = C.expected_face(case, env, scn, normals, k, m, w, h) * factor
        ok_val, ok_sens = C.check_face(acc, m, E, f"shadow veils face {k}", report)
        bad += [] if (ok_val and ok_sens) else [k]
    print("\n".join(report))
    assert not bad, "\n".join(report)
