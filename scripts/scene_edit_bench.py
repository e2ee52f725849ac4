#!/usr/bin/env python
"""Time the scene edits against a full b200pt_set_scene on SynthSponza (the bench.py scene) at 1080p.

Each number is a host clock around one synchronous call (every edit entry point waits for the device before it returns),
median of --reps calls after one warm-up call.  Edits: an in-place material edit (base colour of one opaque material), a
variant-style swap of two opaque render nodes' materials, and a visibility toggle of one render node (a tree rebuild) with
each BVH builder.  The card's name and power limit are printed by the same run.

    python scripts/scene_edit_bench.py [--reps 5] [--tex 2048]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def timed(fn, reps):
    fn()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--tex", type=int, default=2048)
    args = ap.parse_args()
    import numpy as np
    from vk_gltf_renderer_b200 import hdr, synth
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    scn = synth.synth_sponza(seed=1234, tex_size=args.tex)
    env = hdr.load_hdr(os.path.join(ROOT, "tests", "assets", "std_env.hdr"))
    res = Resources(scene=scn, hdr_rgb=env, camera=scn.camera, size=(1920, 1080))
    pt = PathTracer(0)
    pt.onAttach(res)
    pt.ptMaxDepth = 12
    for f in range(2):
        res.frameCount = f
        pt.onRender(None, res)
    pt.synchronize()
    out = dict(gpu=gpu, triangles=scn.num_triangles(), render_nodes=len(scn.render_nodes))
    out["set_scene_ms"] = timed(lambda: pt.onSceneInvalidated(res), args.reps)

    opaque = [i for i, rn in enumerate(scn.render_nodes) if scn.materials[max(0, rn["materialID"])].alphaMode == 0]
    m = scn.materials[max(0, scn.render_nodes[opaque[0]]["materialID"])]

    def material_edit():
        m.pbrBaseColorFactor[0] = 1.0 - m.pbrBaseColorFactor[0]
        pt.update_materials(res)
    out["material_edit_ms"] = timed(material_edit, args.reps)

    a, b = opaque[0], next(i for i in opaque if scn.render_nodes[i]["materialID"] != scn.render_nodes[opaque[0]]["materialID"])

    def node_material_swap():
        ra, rb = scn.render_nodes[a], scn.render_nodes[b]
        ra["materialID"], rb["materialID"] = rb["materialID"], ra["materialID"]
        pt.update_node_materials(res)
    out["node_material_swap_ms"] = timed(node_material_swap, args.reps)

    def toggle():
        rn = scn.render_nodes[opaque[0]]
        rn["visible"] = not rn.get("visible", True)
        pt.set_node_visibility(res)
    for builder in (0, 1):
        pt.set_bvh_builder(builder)
        pt.onSceneInvalidated(res)
        out[f"visibility_toggle_builder{builder}_ms"] = timed(toggle, args.reps)
    pt.onDetach()
    print(json.dumps({k: (round(v, 2) if isinstance(v, float) else v) for k, v in out.items()}))


if __name__ == "__main__":
    main()
