"""-m gpu: the device's tree walks on the families of tests/walkcases.py (nodes far from the origin relative to their size, flat
nodes, slivers, coincident triangles, +-0 and clamped direction components, origins on a surface, segments ending at their hit),
through b200pt_trace_closest / b200pt_trace_shadow, which run the frame's walk sequence (walk, any-hit rounds, continuation walks).

All-opaque scenes: every ray's nearest hit (t, id) equals the kernel-arithmetic brute force bit for bit and every shadow segment is
occluded exactly when the brute force has a hit on it -- with both tree builders, with one and with the default number of
continuation rounds, and again after a node-matrix update moved the scene and refitted the tree.  Non-opaque scenes (alpha blend,
stochastic any-hit): hits, seeds and transmission equal the oracle's bit for bit.  Shadow rays start at t = 0 (see _check).  Rays with a hit whose fp32 t is too
ill-conditioned for the node test's widening (tests/test_walk_precision.py) are left out of the exact comparisons and counted."""
import numpy as np
import pytest

import walkcases as W
from gpu_util import to_dev, trace_both
from test_gpu_scenes import _attach
from test_walk_precision import brute_force, compile_checker

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def checker(tmp_path_factory):
    return compile_checker(tmp_path_factory.mktemp("walkcheck"))


def _device(pt, R):
    import torch
    d_rays = to_dev(R)
    hits = torch.empty((len(R), 6), dtype=torch.float32, device="cuda")
    pt.trace_closest(d_rays.data_ptr(), len(R), hits.data_ptr())
    tr = torch.empty((len(R), 3), dtype=torch.float32, device="cuda")
    pt.trace_shadow(d_rays.data_ptr(), len(R), tr.data_ptr())
    pt.synchronize()
    return hits.cpu().numpy(), tr.cpu().numpy()


def _check(pt, exe, d, tag, v, R, what):
    """closest hits against the brute force of R, shadow rays against the brute force of R from t = 0: b200pt_trace_shadow starts
    every segment at 0, as the frame's shadow rays do (the path state keeps no tmin for them)"""
    bf = brute_force(exe, d, tag, v, R)
    R0 = R.copy()
    R0[:, 3] = 0.0
    bf0 = brute_force(exe, d, tag + "_from0", v, R0)
    hits, tr = _device(pt, R)
    keep = ~np.isin(np.arange(len(R)), np.union1d(bf["ill"], bf0["ill"]))
    got_id = hits.view(np.int32)[:, 3].astype(np.int64)
    want = bf["near_id"] >= 0
    bad_c = (got_id != bf["near_id"]) | (want & (hits[:, 0].view(np.uint32) != bf["near_t"].view(np.uint32)))
    bad_s = (tr[:, 0] == 0) != (bf0["near_id"] >= 0)
    print("%s: closest mismatches %d, shadow %d on %d rays; %d rays with an ill-conditioned hit: %d, %d"
          % (what, (bad_c & keep).sum(), (bad_s & keep).sum(), keep.sum(), (~keep).sum(), (bad_c & ~keep).sum(), (bad_s & ~keep).sum()))
    assert (bad_c & keep).sum() == 0 and (bad_s & keep).sum() == 0
    assert want.mean() > 0.3


@pytest.mark.parametrize("rounds", [1, None])
@pytest.mark.parametrize("builder", [0, 1])
@pytest.mark.parametrize("name", W.FAMILIES)
def test_device_walks_match_brute_force(checker, tmp_path, std_env, monkeypatch, name, builder, rounds):
    from vk_gltf_renderer_b200 import synth
    from vk_gltf_renderer_b200.scene import _glm
    if rounds is not None:
        monkeypatch.setenv("B200PT_CONT_ROUNDS", str(rounds))
    v, R = W.case(name)
    scn = synth.triangle_soup(0, vertices=v, double_sided=1)
    pt, res = _attach(scn, std_env, (16, 16))
    if builder:
        pt.set_bvh_builder(builder)
        pt.onSceneInvalidated(res)
    _check(pt, checker, str(tmp_path), name, v, R, "%s builder %d" % (name, builder))
    # move the scene by 5 % of its extent: b200pt_update_transforms recomputes the triangle records (v + T in fp32, as below) and
    # refits the tree; the rays move along so that they keep their aim
    ext = float((v.reshape(-1, 3).max(0) - v.reshape(-1, 3).min(0)).max())
    T = (np.array([0.05, -0.03, 0.02]) * ext).astype(np.float32)
    m = np.eye(4)
    m[:3, 3] = T
    scn.render_nodes[0]["objectToWorld"] = _glm(m)
    scn.render_nodes[0]["worldToObject"] = _glm(np.linalg.inv(m))
    pt.update_transforms(res)
    R2 = R.copy()
    R2[:, 0:3] = R[:, 0:3] + T
    _check(pt, checker, str(tmp_path), name + "_moved", (v + T).astype(np.float32), R2, "%s builder %d refitted" % (name, builder))
    pt.onDetach()


@pytest.mark.parametrize("rounds", [1, None])
@pytest.mark.parametrize("builder", [0, 1])
@pytest.mark.parametrize("name", ["soup_1e4_at_1e5", "soup_1_at_1e5", "tiny_1e-5", "layers", "duplicates"])
def test_device_walks_match_the_oracle_with_any_hit(checker, tmp_path, std_env, oracle_mod, monkeypatch, name, builder, rounds):
    """alpha-blended (alpha 0.5) soups: every triangle is an any-hit candidate, so the walks run the continuation protocol"""
    from vk_gltf_renderer_b200 import synth
    if rounds is not None:
        monkeypatch.setenv("B200PT_CONT_ROUNDS", str(rounds))
    v, R = W.case(name)
    R[:, 3] = 0.0  # trace_both sends the same rays as shadow rays, and those start at t = 0 on the device (see _check)
    R = R[brute_force(checker, str(tmp_path), name, v, R)["well"]]
    scn = synth.triangle_soup(0, vertices=v, double_sided=1, material=dict(pbrBaseColorFactor=[0.8, 0.8, 0.8, 0.5], alphaMode=2))
    pt, res = _attach(scn, std_env, (16, 16))
    if builder:
        pt.set_bvh_builder(builder)
        pt.onSceneInvalidated(res)
    o = oracle_mod.Oracle()
    o.set_scene(scn)
    seeds = ((np.arange(len(R), dtype=np.uint64) * 2654435761) % (2 ** 32)).astype(np.uint32)
    ref, _, ref_t, _ = trace_both(pt, o, R, seeds, tmax=1e30)
    assert (ref.view(np.int32)[:, 3] >= 0).mean() > 0.2
    pt.onDetach()
