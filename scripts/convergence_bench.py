"""Convergence against plain frames: SynthSponza at 1920x1080, depth 12, 1 spp per frame, rendered with b200pt_set_convergence at
thresholds 0.05 / 0.02 / 0.01 (minFrames 16, interval 8, at most 256 frames) and without it up to the same last frame.

Both loops read the image state at every checkpoint (the convergence run its active-pixel count, the plain run its image), so both
synchronise equally often; the GPU time of the frames is taken with CUDA events on the handle's stream around each block of `interval`
frames, excluding the reads.  Prints one JSON line per threshold with:
  - frames, GPU ms and pathsStarted of the convergence run and of the plain run to the same last frame;
  - the share of pixels active at each checkpoint;
  - the mean relative luminance error of both images against a long plain render, at equal GPU time (the plain image is the one after
    the last block that ended within the convergence run's time);
then one line with the mechanism's overhead alone (threshold 1e-9: nothing stops) against plain frames, alternated, and the card name,
power limit and maximum SM clock read in the same run.

    python scripts/convergence_bench.py [--thresholds 0.05,0.02,0.01] [--max-frames 256] [--ref-frames 1024] [--size 1920x1080]
"""
import argparse
import json
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
    ap.add_argument("--thresholds", default="0.05,0.02,0.01")
    ap.add_argument("--max-frames", type=int, default=256)
    ap.add_argument("--ref-frames", type=int, default=1024, help="frames of the long plain render the errors are taken against")
    ap.add_argument("--min-frames", type=int, default=16)
    ap.add_argument("--interval", type=int, default=8)
    ap.add_argument("--size", default="1920x1080")
    ap.add_argument("--depth", type=int, default=12)
    ap.add_argument("--tex", type=int, default=2048)
    ap.add_argument("--overhead-frames", type=int, default=64)
    ap.add_argument("--overhead-rounds", type=int, default=3)
    args = ap.parse_args()

    import torch
    from vk_gltf_renderer_b200 import camera, hdr, synth
    from vk_gltf_renderer_b200.renderer import PathTracer, Resources
    if not torch.cuda.is_available():
        sys.exit("convergence_bench.py measures on the GPU; no CUDA device is visible")
    w, h = (int(x) for x in args.size.split("x"))
    scn = synth.synth_sponza(seed=1234, tex_size=args.tex)
    env = hdr.load_hdr(os.path.join(ROOT, "tests", "assets", "std_env.hdr"))
    res = Resources(scene=scn, hdr_rgb=env, camera=scn.camera, size=(w, h))
    pt = PathTracer(0)
    pt.ptMaxDepth = args.depth
    pt.onAttach(res)
    stream = torch.cuda.ExternalStream(pt.stream())
    fi = camera.make_frame_info(scn.camera, w, h)
    pcs = [camera.make_push_constant(scn.camera, h, frame_count=f, total_samples=f, num_samples=1, max_depth=args.depth)
           for f in range(max(args.ref_frames, args.max_frames))]

    def lum(img):
        return img[..., :3].astype(np.float64).mean(-1)

    def run(frames, on_block):
        """renders frames 0..frames-1 in blocks of `interval`; on_block(F) after each block (outside the timed region) may end the run.
        Returns (frames rendered, GPU ms, pathsStarted)."""
        pt.synchronize()
        pt.reset_stats()
        ms, f = 0.0, 0
        while f < frames:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(stream)
            for _ in range(min(args.interval, frames - f)):
                pt.render_frame_raw(fi, pcs[f])
                f += 1
            pt.flush()
            b.record(stream)
            b.synchronize()
            ms += a.elapsed_time(b)
            if on_block(f, ms):
                break
        return f, ms, pt.stats()["pathsStarted"]

    pt.set_convergence(0)
    run(8, lambda f, ms: False)  # warm-up
    run(args.ref_frames, lambda f, ms: False)
    ref = lum(pt.read_accum())

    def rel_err(img):
        return float(np.mean(np.abs(lum(img) - ref) / np.maximum(ref, 1e-3)))

    plain_trace = []  # (frames, ms, error) after every block of a plain run to max_frames
    run(args.max_frames, lambda f, ms: plain_trace.append((f, ms, rel_err(pt.read_accum()))) and False)
    for thr in (float(t) for t in args.thresholds.split(",")):
        pt.set_convergence(thr, floor=1e-3, min_frames=args.min_frames, interval=args.interval)
        active = []

        def block(f, ms):
            active.append(pt.read_convergence()[2])
            return active[-1] == 0

        frames, ms, started = run(args.max_frames, block)
        err = rel_err(pt.read_accum())
        pt.set_convergence(0)
        pf, pms, pstarted = run(frames, lambda f, ms: False)
        eq = [t for t in plain_trace if t[1] <= ms]
        print(json.dumps({"threshold": thr, "frames": frames, "ms": round(ms, 2), "paths_started": started, "plain_ms": round(pms, 2),
                          "plain_paths_started": pstarted, "speedup": round(pms / ms, 3),
                          "active_share_at_checkpoints": [round(a / (w * h), 4) for a in active],
                          "rel_error": round(err, 5), "plain_rel_error_at_equal_time": round(eq[-1][2], 5) if eq else None,
                          "plain_frames_at_equal_time": eq[-1][0] if eq else 0}), flush=True)

    # the mechanism alone: nothing stops, so the convergence run traces every path the plain run traces
    # (the convergence run reads its active count at every checkpoint, as a caller ending its loop would)
    conv_ms, plain_ms = [], []
    for _ in range(args.overhead_rounds):
        pt.set_convergence(1e-9, floor=1e-3, min_frames=args.min_frames, interval=args.interval)
        conv_ms.append(run(args.overhead_frames, lambda f, ms: pt.read_convergence()[2] == 0)[1])
        pt.set_convergence(0)
        plain_ms.append(run(args.overhead_frames, lambda f, ms: False)[1])
    if conv_ms:
        print(json.dumps({"overhead_frames": args.overhead_frames, "conv_ms": [round(x, 2) for x in conv_ms], "plain_ms": [round(x, 2) for x in plain_ms],
                          "overhead": round(sum(conv_ms) / sum(plain_ms) - 1.0, 4)}), flush=True)
    print(json.dumps({"card": card()}), flush=True)
    pt.onDetach()


if __name__ == "__main__":
    main()
