"""Views against separate frames: SynthSponza at depth 12, 1 spp, V camera poses rendered as ONE b200pt_render_views call against the
same V poses as V b200pt_render_frame calls, on one handle, at 256x256, 512x512 and 1920x1080.  The two are timed alternately in one
process, after a warm-up, with CUDA events on the handle's stream around a block of frames that starts and ends with the device idle.
Prints one JSON line per (size, V) with Mray/s of each and their ratio, then the card name, power limit and maximum SM clock read
in the same run.

    python scripts/views_bench.py [--views 1,2,6,16] [--sizes 256x256,512x512,1920x1080] [--rounds 3] [--frames 2] [--tex 2048]
"""
import argparse
import json
import math
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                         timeout=30).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--views", default="1,2,6,16")
    ap.add_argument("--sizes", default="256x256,512x512,1920x1080")
    ap.add_argument("--rounds", type=int, default=3, help="timed blocks of each variant, alternated")
    ap.add_argument("--frames", type=int, default=2, help="frames per timed block")
    ap.add_argument("--depth", type=int, default=12)
    ap.add_argument("--tex", type=int, default=2048)
    ap.add_argument("--lanes", type=int, default=4, help="frames in flight")
    args = ap.parse_args()

    import torch
    from vk_gltf_renderer_b200 import camera, hdr, synth
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    if not torch.cuda.is_available():
        sys.exit("views_bench.py measures on the GPU; no CUDA device is visible")
    scn = synth.synth_sponza(seed=1234, tex_size=args.tex)
    env = hdr.load_hdr(os.path.join(ROOT, "tests", "assets", "std_env.hdr"))
    sizes = [tuple(int(x) for x in s.split("x")) for s in args.sizes.split(",")]
    res = Resources(scene=scn, hdr_rgb=env, camera=scn.camera, size=sizes[0])
    pt = PathTracer(0)
    pt.ptMaxDepth = args.depth
    pt.onAttach(res)
    pt.set_frames_in_flight(args.lanes)
    stream = torch.cuda.ExternalStream(pt.stream())
    cam = scn.camera
    eye, center = np.asarray(cam.eye, np.float64), np.asarray(cam.center, np.float64)
    frame = [0]

    def timed(render):
        """Mray/s of args.frames frames through render(pc)"""
        pt.synchronize()
        pt.reset_stats()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        for _ in range(args.frames):
            f = frame[0]
            frame[0] += 1
            render(camera.make_push_constant(cam, res.size[1], frame_count=f, total_samples=f, num_samples=1, max_depth=args.depth))
        pt.flush()
        e1.record(stream)
        e1.synchronize()
        st = pt.stats()
        return (st["closestRays"] + st["shadowRays"]) / (e0.elapsed_time(e1) * 1e3)

    rows = []
    for w, h in sizes:
        for nv in (int(v) for v in args.views.split(",")):
            pt.set_views(1)
            pt.onResize(None, (w, h), res)
            pt.set_views(nv)
            base = camera.make_frame_info(cam, w, h)
            poses = []
            for k in range(nv):  # a turntable ring about the look-at point, 2 degrees apart
                a = math.radians(2.0 * k)
                rot = np.array([[math.cos(a), 0.0, math.sin(a)], [0.0, 1.0, 0.0], [-math.sin(a), 0.0, math.cos(a)]])
                poses.append(camera.look_at(center + rot @ (eye - center), center, cam.up))
            fis = camera.view_frame_infos(base, poses)
            variants = {"views": lambda pc: pt.render_views(fis, pc),
                        "frames": lambda pc: [pt.render_frame_raw(fi, pc) for fi in fis]}
            frame[0] = 0
            for render in variants.values():  # warm-up of both
                timed(render)
            rate = {k: [] for k in variants}
            for _ in range(args.rounds):
                for k, render in variants.items():
                    rate[k].append(timed(render))
            row = {"size": f"{w}x{h}", "views": nv, "paths_per_call": w * h * nv,
                   "mray_s_views": round(float(np.median(rate["views"])), 1), "mray_s_frames": round(float(np.median(rate["frames"])), 1),
                   "spread_views": [round(min(rate["views"]), 1), round(max(rate["views"]), 1)],
                   "spread_frames": [round(min(rate["frames"]), 1), round(max(rate["frames"]), 1)]}
            row["speedup"] = round(row["mray_s_views"] / row["mray_s_frames"], 3)
            rows.append(row)
            print(json.dumps(row), flush=True)
    pt.onDetach()
    print(json.dumps({"card": card(), "depth": args.depth, "frames_in_flight": args.lanes, "frames_per_block": args.frames,
                      "rounds": args.rounds}), flush=True)


if __name__ == "__main__":
    main()
