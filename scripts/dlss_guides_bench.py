"""Cost of the DLSS variant: SynthSponza at 1080p, depth 12, one sample per frame, plain frames and DLSS frames (Halton jitter,
six guide images, a slowly moving camera) alternated in one process on one GPU.  Prints one JSON line with ms per frame and
Mray/s of each variant, and the card and power limit read in the same run.

    python scripts/dlss_guides_bench.py [--frames 20] [--rounds 3] [--width 1920 --height 1080] [--tex 2048]

Frames are unbatched in both variants (a DLSS frame never joins a frame batch); timing is the host clock around a block of
frames that ends in a device synchronise.
"""
import argparse
import copy
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return out[0] if out else "unknown"
    except (OSError, subprocess.TimeoutExpired):
        return "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--depth", type=int, default=12)
    ap.add_argument("--tex", type=int, default=2048)
    args = ap.parse_args()
    from vk_gltf_renderer_b200 import hdr, synth
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    scn = synth.synth_sponza(seed=1234, tex_size=args.tex)
    env = hdr.load_hdr(os.path.join(ROOT, "tests", "assets", "std_env.hdr"))
    res = Resources(scene=scn, hdr_rgb=env, camera=scn.camera, size=(args.width, args.height))
    pt = PathTracer(0)
    pt.ptMaxDepth = args.depth
    pt.ptSamples = 1
    pt.onAttach(res)
    pt.set_frame_batch(1)
    cam0 = scn.camera

    def block(dlss):
        pt.set_dlss_guides(dlss)
        pt.synchronize()
        pt.reset_stats()
        t0 = time.perf_counter()
        for f in range(args.frames):
            cam = copy.deepcopy(cam0)
            cam.eye = (np.asarray(cam0.eye, np.float64) + np.array([0.002 * f, 0, 0])).astype(np.float32) if dlss else cam0.eye
            res.camera = cam
            res.frameCount = f
            pt.onRender(None, res)
        pt.synchronize()
        dt = time.perf_counter() - t0
        st = pt.stats()
        return dt * 1e3 / args.frames, (st["closestRays"] + st["shadowRays"]) / dt / 1e6

    block(False)
    block(True)   # warm-up of both variants
    runs = {"plain": [], "dlss": []}
    for _ in range(args.rounds):
        for name, dlss in (("plain", False), ("dlss", True)):
            runs[name].append(block(dlss))
    line = {"scene": "SynthSponza(seed=1234) %dx%d, depth %d, 1 spp per frame, unbatched" % (args.width, args.height, args.depth), "card": card(),
            "frames_per_round": args.frames, "rounds": args.rounds}
    for name, r in runs.items():
        line[name] = {"ms_per_frame": [round(x[0], 3) for x in r], "mray_s": [round(x[1], 1) for x in r]}
    print(json.dumps(line))
    pt.onDetach(res)


if __name__ == "__main__":
    main()
