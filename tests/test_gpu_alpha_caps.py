"""-m gpu alpha caps (csrc/alpha_caps.cuh): a candidate whose micro-triangle is opaque everywhere passes its any-hit test whatever it
draws, so the walks stop looking behind it.  A handle with caps must answer exactly what a handle without them (B200PT_ALPHA_CAPS=0)
answers: the ray-level API's hits (t, u, v, id), seeds and transmission, and the accumulation, selection and ray counters of frames,
bit for bit.  The traversal-counter build shows that the caps were there: the walks with caps test fewer triangles."""
import numpy as np
import pytest

from gpu_util import random_rays, to_dev
from test_gpu_scene_edits import _assert_same, _clone, _render

pytestmark = pytest.mark.gpu

SIZE = (96, 72)
STATS = ("closestRays", "shadowRays", "shadedHits", "pathsStarted")


def _handle(scn, env, caps, monkeypatch, count=False, depth=5):
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    monkeypatch.setenv("B200PT_ALPHA_CAPS", "1" if caps else "0")
    res = Resources(scene=scn, hdr_rgb=env, camera=scn.camera, size=SIZE)
    pt = PathTracer(0, count_traversal=count)
    pt.ptMaxDepth = depth
    pt.onAttach(res)
    return pt, res


def _rays(pt, rays, seeds, tmax):
    """closest-hit rays, then the same rays as shadow rays cut at tmax: hits, transmission and both seed arrays"""
    import torch
    d_seeds = [to_dev(seeds.copy()), to_dev(seeds.copy())]
    hits = torch.empty((len(rays), 6), dtype=torch.float32, device="cuda")
    pt.trace_closest(to_dev(rays).data_ptr(), len(rays), hits.data_ptr(), d_seeds[0].data_ptr())
    rs = rays.copy()
    rs[:, 7] = tmax
    trans = torch.empty((len(rays), 3), dtype=torch.float32, device="cuda")
    pt.trace_shadow(to_dev(rs).data_ptr(), len(rs), trans.data_ptr(), d_seeds[1].data_ptr())
    pt.synchronize()
    return dict(hits=hits.cpu().numpy(), trans=trans.cpu().numpy(), seeds=np.stack([s.cpu().numpy() for s in d_seeds]))


def _snapshot(pt, res, rays, seeds, tmax):
    pt.reset_stats()
    _render(pt, res)
    out = dict(img=pt.read_accum())
    out["ids"], out["depth"] = pt.read_selection()
    st = pt.stats()
    out["stats"] = [st[k] for k in STATS]
    out.update(_rays(pt, rays, seeds, tmax))
    return out


def _seeds(n, mul=2654435761):
    return ((np.arange(n, dtype=np.uint64) * mul) % (2 ** 32)).astype(np.uint32)


def _deep_layers():
    """14 MASK layers (noise alpha with opaque regions) without micromaps, two of them mirrored, and rays through all of them"""
    from vk_gltf_renderer_b200 import synth
    from vk_gltf_renderer_b200.scene import _glm
    scn = synth.synth_layers(tex_size=256)
    for rn in scn.render_nodes[2:4]:
        m = np.asarray(rn["objectToWorld"], np.float64).reshape(4, 4).T.copy() @ np.diag([-1.0, 1.0, 1.0, 1.0])
        rn["objectToWorld"], rn["worldToObject"] = _glm(m), _glm(np.linalg.inv(m))
    rng = np.random.default_rng(11)
    n = 40000
    rays = np.zeros((n, 8), np.float32)
    rays[:, 0:3] = np.stack([rng.uniform(-1.4, 1.4, n), rng.uniform(0.2, 2.0, n), rng.uniform(0.5, 3.0, n)], 1)
    tgt = np.stack([rng.uniform(-1.4, 1.4, n), rng.uniform(0.2, 2.0, n), np.full(n, -2.4)], 1)
    d = tgt - rays[:, 0:3]
    rays[:, 4:7] = d / np.linalg.norm(d, axis=1, keepdims=True)
    rays[:, 7] = 1e32
    return scn, rays, _seeds(n, 40503), 0.7


def _case(name):
    from vk_gltf_renderer_b200 import synth
    if name == "atrium":
        rays = random_rays(60000, [-15, 0, -6], [15, 12, 6])
        return synth.synth_sponza(tex_size=256, detail=0.05), rays, _seeds(len(rays)), 4.0
    if name == "tinted_layers":
        # glass sheets: non-opaque only through transmission (alpha mode OPAQUE), so every micro-triangle caps closest-hit rays and
        # none caps a shadow ray (transmission 0.9)
        rays = random_rays(40000, [-1.6, 0.1, -2.2], [1.9, 2.1, 3.0])
        return synth.synth_layers(tinted=True), rays, _seeds(len(rays)), 4.0
    if name == "sampler_layers":
        # clamped, mirrored, nearest, non-power-of-two, N x 1, vertex-colour alpha, spec-gloss and BLEND layers
        rays = random_rays(60000, [-1.6, 0.1, -2.2], [1.9, 2.1, 0.2])
        return synth.sampler_layers(), rays, _seeds(len(rays)), 4.0
    return _deep_layers()


def _draws(seed_in, seed_out, most=64):
    """how many rnd() a ray drew: pcg steps (vec.cuh) from its seed before the call to its seed after it"""
    s, out = seed_in.astype(np.uint64), np.full(len(seed_in), -1)
    for k in range(most + 1):
        out[(out < 0) & (s == seed_out)] = k
        s = (s * 747796405 + 2891336453) % (1 << 32)
    assert (out >= 0).all()
    return out


def _tris_tested(scn, env, caps, rays, seeds, tmax, monkeypatch):
    pt, _ = _handle(scn, env, caps, monkeypatch, count=True)
    pt.reset_stats()
    _rays(pt, rays, seeds, tmax)
    n = pt.stats()["trisTested"]
    pt.onDetach()
    return n


# rounds = 1: rays behind more than 2 x 4 rejected candidates finish in the in-kernel fallback of the last k_alpha, with caps behind them
@pytest.mark.parametrize("rounds", [1, 2])
@pytest.mark.parametrize("case", ["atrium", "sampler_layers", "tinted_layers", "deep_layers"])
def test_caps_change_no_result(std_env, monkeypatch, case, rounds):
    monkeypatch.setenv("B200PT_CONT_ROUNDS", str(rounds))
    scn, rays, seeds, tmax = _case(case)
    out = []
    for caps in (True, False):
        pt, res = _handle(_clone(scn), std_env, caps, monkeypatch)
        out.append(_snapshot(pt, res, rays, seeds, tmax))
        pt.onDetach()
    _assert_same(out[0], out[1], case)
    # the deep stack lets some shadow rays through and blocks others; closest-hit rays that draw 5-8 times finished in a continuation
    # round, more than 4 + 4 R in the in-kernel fallback of the last k_alpha -- both with caps behind the rejected candidates
    if case == "deep_layers":
        assert 0.02 < (out[0]["trans"][:, 0] > 0).mean() < 0.98
        d = _draws(seeds, out[0]["seeds"][0])
        assert ((d > 4) & (d <= 4 + 4 * rounds)).sum() > 500 and (d > 4 + 4 * rounds).sum() > 50, np.bincount(d)
    with_caps, without = (_tris_tested(_clone(scn), std_env, c, rays, seeds, tmax, monkeypatch) for c in (True, False))
    assert with_caps < without, (case, with_caps, without)


def test_cutoff_edit_rebakes_the_caps(std_env, monkeypatch):
    """b200pt_update_materials in place moves the MASK cutoff up and down, then changes only the roughness: the edited handle with caps
    renders and traces what a fresh handle without caps renders and traces (a stale map would stop walks at texels that are no longer
    opaque)."""
    scn, rays, seeds, tmax = _deep_layers()
    pt, res = _handle(scn, std_env, True, monkeypatch)
    _render(pt, res)
    # the last step changes no alpha input (the caps stay as they are)
    for cutoff, roughness in ((0.95, None), (1.0, None), (0.2, None), (0.5, None), (0.5, 0.35)):
        for m in res.scene.materials:
            if m.alphaMode == 1:
                m.alphaCutoff = cutoff
                if roughness is not None:
                    m.pbrRoughnessFactor = roughness
        monkeypatch.setenv("B200PT_ALPHA_CAPS", "1")
        pt.update_materials(res)
        got = _snapshot(pt, res, rays, seeds, tmax)
        ref_pt, ref_res = _handle(_clone(res.scene), std_env, False, monkeypatch)
        _assert_same(got, _snapshot(ref_pt, ref_res, rays, seeds, tmax), cutoff)
        ref_pt.onDetach()
    pt.onDetach()
