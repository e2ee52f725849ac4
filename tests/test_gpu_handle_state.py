"""-m gpu: what a handle holds after a call it refused.  A refused scene leaves no scene behind, so b200pt_render_frame refuses until
the next valid scene, and that scene renders on the handle exactly as on a fresh one."""
import numpy as np
import pytest

from test_gpu_materials import malformed_scenes
from test_gpu_omm import micromap_scene_and_bad_sets

pytestmark = pytest.mark.gpu


def test_refused_scenes_leave_no_scene_behind(box_scene, std_env):
    from vk_gltf_renderer_b200.renderer import B200PTError, PathTracer, Resources, render_headless
    size = (48, 32)
    res = Resources(scene=box_scene, hdr_rgb=std_env, camera=box_scene.camera, size=size)
    pt = PathTracer(0)
    pt.onAttach(res)

    def refused(scn):
        with pytest.raises(B200PTError):
            pt.onSceneInvalidated(Resources(scene=scn, hdr_rgb=std_env, camera=scn.camera, size=size))
        res.frameCount = 0
        with pytest.raises(B200PTError, match="set_scene and resize must come first"):
            pt.onRender(None, res)

    for _, scn in malformed_scenes(box_scene):
        refused(scn)
    layers, bad = micromap_scene_and_bad_sets()
    for b in bad:
        layers.micromaps, layers.prim_omms = b["mm"], b["po"]
        refused(layers)
    layers.micromaps, layers.prim_omms = [], []
    here = Resources(scene=layers, hdr_rgb=std_env, camera=layers.camera, size=size)
    pt.onSceneInvalidated(here)
    _, img = render_headless(here, 3, pt=pt)
    _, fresh = render_headless(Resources(scene=layers, hdr_rgb=std_env, camera=layers.camera, size=size), 3)
    assert np.array_equal(img.view(np.uint32), fresh.view(np.uint32))
    assert img[..., 3].max() > 0
    pt.onDetach()
