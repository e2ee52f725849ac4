"""-m gpu: the DLSS variant (b200pt_set_dlss_guides / b200pt_read_dlss_guides) against the oracle over four DLSS frames with Halton
jitters, a moving camera and one node update between frames 2 and 3, on the textured material zoo, the shadow-catcher scene
(driven through the device node hierarchy) and SynthGlass; then the frame scheduling (frames in flight, frame batching, an
interleaved tile) and the combination with the OptiX guide image."""
import copy
import math

import numpy as np
import pytest

from conftest import rel_rmse

pytestmark = pytest.mark.gpu
W, H = 128, 96
FRAMES = 4


def _camera_at(cam0, f):
    cam = copy.deepcopy(cam0)
    a = 0.03 * f
    off = np.asarray(cam.eye, np.float64) - np.asarray(cam.center, np.float64)
    rot = np.array([[math.cos(a), 0, math.sin(a)], [0, 1, 0], [-math.sin(a), 0, math.cos(a)]])
    cam.eye = (np.asarray(cam.center, np.float64) + rot @ off + np.array([0.02 * f, 0.01 * f, 0])).astype(np.float32)
    return cam


def _moved(scn, node, shift):
    from vk_gltf_renderer_b200 import synth
    out = synth.scene_from_state(copy.deepcopy(synth.scene_state(scn)))
    m = np.asarray(out.render_nodes[node]["objectToWorld"], np.float64).reshape(4, 4).T
    m[:3, 3] += shift
    out.render_nodes[node]["objectToWorld"] = np.ascontiguousarray(m.T.reshape(16), np.float32)
    out.render_nodes[node]["worldToObject"] = np.ascontiguousarray(np.linalg.inv(m).T.reshape(16), np.float32)
    return out


def _o2w(scn):
    return np.stack([np.asarray(rn["objectToWorld"], np.float32) for rn in scn.render_nodes])


class Case:
    """scene + how the node update between frames 2 and 3 happens, on the device (pt) and for the oracle (scene, prev o2w)"""

    def __init__(self, kind, std_env):
        from vk_gltf_renderer_b200 import synth
        self.settings = {}
        self.hier = None
        if kind == "zoo":
            self.scn = synth.synth_material_zoo()
            self.scn2 = _moved(self.scn, 1, [0.15, 0.05, -0.1])
        elif kind == "glass":
            self.scn = synth.synth_glass()
            self.scn2 = _moved(self.scn, 0, [0.1, 0.0, 0.08])
        else:   # shadow catcher on the lit scene, its nodes driven by the device hierarchy
            from oracle import animation as A
            from vk_gltf_renderer_b200.animation import topo_levels
            scn, parents, mappings, inst, pose = synth.synth_hierarchy()
            glm = lambda ms: np.ascontiguousarray(np.asarray(ms, np.float64).transpose(0, 2, 1).astype(np.float32))
            order, offsets = topo_levels(parents)
            scenes = []
            for k in (0, 1):
                o2w, w2o = A.render_nodes(A.propagate(glm(pose(k)), parents, order, offsets), mappings, glm(inst))
                s = synth.scene_from_state(copy.deepcopy(synth.scene_state(scn)))
                for i, rn in enumerate(s.render_nodes):
                    rn["objectToWorld"], rn["worldToObject"] = o2w[i].reshape(-1).copy(), w2o[i].reshape(-1).copy()
                scenes.append(s)
            self.scn, self.scn2 = scenes
            self.hier = (scn, parents, mappings, glm(inst), [glm(pose(0)), glm(pose(1))])
            # the catcher plane 2 cm above the floor: a plane coplanar with the floor would make every floor pixel an fp32 tie
            self.settings = dict(useInfinitePlane=True, isShadowCatcher=True, infinitePlaneDistance=0.02, shadowCatcherDarkness=0.35)
        self.env = std_env

    def attach(self, lanes=4, batch=1, tile=None, optix=False):
        from vk_gltf_renderer_b200.renderer import PathTracer, Resources
        res = Resources(scene=self.hier[0] if self.hier else self.scn, hdr_rgb=self.env, camera=self.scn.camera, size=(W, H), tile=tile)
        for k, v in self.settings.items():
            setattr(res.settings, k, v)
        pt = PathTracer(0)
        pt.ptMaxDepth = 5
        pt.onAttach(res)
        pt.set_frames_in_flight(lanes)
        pt.set_frame_batch(batch)
        if self.hier:
            _, parents, mappings, inst, locs = self.hier
            pt.set_node_hierarchy(parents, mappings, inst)
            pt.update_node_matrices(locs[0])
        if optix:
            pt.set_guide_outputs(True)
        pt.set_dlss_guides(True)
        return pt, res

    def update(self, pt, res):
        if self.hier:
            pt.update_node_matrices(self.hier[4][1])
        else:
            res.scene = self.scn2
            pt.update_transforms(res)

    def run_device(self, **kw):
        pt, res = self.attach(**kw)
        out = []
        for f in range(FRAMES):
            if f == 2:
                self.update(pt, res)
            res.camera = _camera_at(self.scn.camera, f)
            res.frameCount = f
            pt.onRender(None, res)
            g = pt.read_dlss_guides()
            g["image"] = pt.read_accum()
            if kw.get("optix"):
                g["optix_albedo"], g["optix_normal"] = pt.read_guide()
            out.append(g)
        pt.onDetach(res)
        return out

    def run_oracle(self, oracle_mod, optix=False):
        from vk_gltf_renderer_b200 import abi, camera as camm
        o = oracle_mod.Oracle()
        o.set_environment(self.env)
        o.set_scene(self.scn)
        s = self.settings
        accum = np.zeros((H, W, 4), np.float32)
        prev_vp, out = None, []
        for f in range(FRAMES):
            prev = None
            if f == 2:
                o.set_scene(self.scn2)
                prev = _o2w(self.scn)
            cam = _camera_at(self.scn.camera, f)
            fi = camm.make_frame_info(cam, W, H, infinite_plane=s.get("useInfinitePlane", False), shadow_catcher=s.get("isShadowCatcher", False),
                                      plane_distance=s.get("infinitePlaneDistance", 0.0), catcher_darkness=s.get("shadowCatcherDarkness", 0.0))
            if prev_vp is not None:
                fi.prevMVP[:] = prev_vp
            prev_vp = list(fi.viewProjMatrix)
            fi.jitter[:] = list(camm.dlss_jitter(f + 1))
            pc = camm.make_push_constant(cam, H, frame_count=f, total_samples=f, num_samples=1, max_depth=5)
            pc.frameCount = f + 1
            pc.flags |= abi.PT_USE_DLSS | (abi.PT_USE_OPTIX_DENOISER if optix else 0)
            guide = np.zeros((H, W, 4), np.float32) if optix else None
            g = o.render_frame_dlss(fi, pc, accum, prev_object_to_world=prev, guide=guide)
            g["image"] = accum.copy()
            if optix:
                g["optix_albedo"], g["optix_normal"] = guide[..., :3].copy(), guide[..., 3].copy().view(np.uint32)
            out.append(g)
        return out


def _check_planes(got, ref, tag):
    for name in ("albedo", "spec_albedo", "normal_roughness", "motion", "depth", "spec_hit_dist"):
        a, b = got[name], ref[name]
        # bit patterns: NaN motion (the lit catcher plane as the first surface keeps the 1e34 first-hit sentinel) compares equal
        eq = a.view(np.uint16 if a.dtype == np.float16 else a.dtype) == b.view(np.uint16 if b.dtype == np.float16 else b.dtype)
        same = eq if a.ndim == 2 else eq.all(-1)
        assert same.mean() > 0.995, (tag, name, same.mean())
        da, db = a.astype(np.float64), b.astype(np.float64)
        finite = np.isfinite(db) & np.isfinite(da)
        da, db = np.where(finite, da, 0.0), np.where(finite, db, 0.0)
        assert np.array_equal(np.isfinite(da), np.isfinite(db)), (tag, name)
        if name == "albedo":
            assert np.abs(da - db).max() <= 1, (tag, name)                       # one UNORM8 step at a rounding boundary
        elif name == "motion":
            assert np.all(np.abs(da - db)[finite] <= 1e-2), (tag, name)
        else:
            assert np.all(np.abs(da - db)[finite] <= 2e-3 * np.abs(db)[finite] + 1e-6), (tag, name)


@pytest.mark.parametrize("kind", ["zoo", "catcher", "glass"])
def test_dlss_frames_match_the_oracle(kind, std_env, oracle_mod):
    case = Case(kind, std_env)
    dev = case.run_device()
    ref = case.run_oracle(oracle_mod)
    for f, (d, r) in enumerate(zip(dev, ref)):
        tag = f"{kind} frame {f}"
        e = rel_rmse(d["image"], r["image"])
        assert e <= 1e-3, (tag, e)
        w_same = (d["image"][..., 3] == r["image"][..., 3]).mean()
        if kind == "catcher":
            # .w is pt.solid, which a shadow-catcher continuation that leaves the scene clears: a path that diverges at the ulp level
            # (what the image tolerance allows for) can flip it
            assert w_same > 0.999, (tag, w_same)
        else:
            assert w_same == 1.0, (tag, w_same)
        _check_planes(d, r, tag)
    moving = np.nanmax(np.abs(np.where(np.isfinite(dev[2]["motion"]), dev[2]["motion"], 0).astype(np.float64)))
    assert moving > 0.1, kind                           # the camera and the updated node moved


def test_dlss_scheduling_is_bit_identical(std_env):
    case = Case("zoo", std_env)
    ref = case.run_device(lanes=1, batch=1)

    def same(a, b, tag):
        for k in ref[0]:
            assert np.array_equal(np.ascontiguousarray(a[k]).view(np.uint8), np.ascontiguousarray(b[k]).view(np.uint8)), (tag, k)
    for lanes, batch in ((4, 1), (1, 3), (4, 3)):
        for f, (a, b) in enumerate(zip(case.run_device(lanes=lanes, batch=batch), ref)):
            same(a, b, (lanes, batch, f))
    band = 8
    ranks = [case.run_device(tile=("interleave", band, 2, r)) for r in (0, 1)]
    for f in range(FRAMES):
        full = {}
        for k in ref[f]:
            full[k] = np.empty_like(ref[f][k])
            for r in (0, 1):
                part = ranks[r][f][k]
                for l0 in range(0, part.shape[0], band):
                    g0 = ((l0 // band) * 2 + r) * band
                    full[k][g0:g0 + band] = part[l0:l0 + band]
        # an interleaved tile sees the same frame but its own image size is the full one: every plane is that of the full frame
        same(full, ref[f], ("interleaved", f))


def test_dlss_with_optix_guides_and_back_to_the_plain_variant(std_env, oracle_mod):
    from vk_gltf_renderer_b200 import abi, camera as camm
    from vk_gltf_renderer_b200.renderer import B200PTError, PathTracer, Resources
    case = Case("zoo", std_env)
    dlss_only = case.run_device()
    both = case.run_device(optix=True)
    ref = case.run_oracle(oracle_mod, optix=True)
    for f in range(FRAMES):
        for k in dlss_only[f]:
            assert np.array_equal(both[f][k], dlss_only[f][k]), (f, k)
        same = (both[f]["optix_albedo"] == ref[f]["optix_albedo"]).all(-1)
        assert same.mean() > 0.995 and (both[f]["optix_normal"] == ref[f]["optix_normal"]).mean() > 0.99, f
    # refusals, then DLSS off: the plain variant, bit-identical to a handle that never had the DLSS guides
    pt, res = case.attach()
    fi = camm.make_frame_info(case.scn.camera, W, H)
    pc = camm.make_push_constant(case.scn.camera, H, frame_count=0, total_samples=0, num_samples=2, max_depth=5)
    pc.flags |= abi.PT_USE_DLSS
    with pytest.raises(B200PTError):
        pt.render_frame_raw(fi, pc)                     # numSamples must be 1
    plain = PathTracer(0)
    plain.ptMaxDepth = 5
    plain.onAttach(Resources(scene=case.scn, hdr_rgb=std_env, camera=case.scn.camera, size=(W, H)))
    pc.numSamples = 1
    with pytest.raises(B200PTError):
        plain.render_frame_raw(fi, pc)                  # no DLSS guides on this handle
    res.frameCount = 0
    pt.onRender(None, res)
    pt.set_dlss_guides(False)
    with pytest.raises(B200PTError):
        pt.read_dlss_guides()
    pt.ptSamples = plain.ptSamples = 2
    res2 = Resources(scene=case.scn, hdr_rgb=std_env, camera=case.scn.camera, size=(W, H))
    for f in range(3):
        res.frameCount = res2.frameCount = f
        pt.onRender(None, res)
        plain.onRender(None, res2)
    assert np.array_equal(pt.read_accum(), plain.read_accum())
    pt.onDetach(res)
    plain.onDetach(res2)
