"""Per-bounce queue sizes and kernel times of the bench workload (tuning aid; needs a GPU)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ["B200PT_DUMP_ITERS"] = "1"
import bench
from vk_gltf_renderer_b200.renderer import PathTracer, Resources

sys.argv = sys.argv[:1]
args = bench.parse()
H = int(os.environ.get("ROWS", args.height))
scn, env = bench.build_workload(args)
res = Resources(scene=scn, hdr_rgb=env, camera=scn.camera, size=(args.width, args.height), tile=(0, H))
pt = PathTracer(0)
pt.ptMaxDepth = args.depth
pt.onAttach(res)
for f in range(4):
    res.frameCount = f
    if f == 3:
        pt.set_profiling(True)
    pt.onRender(None, res)
pt.synchronize()
# the profiled frame's per-stage totals: each stage's column of the per-bounce rows above adds up to these
st = pt.stats()
print("frame totals:", "  ".join(f"{k} {st[k]:.3f}" for k in ("msTraceClosest", "msAnyHit", "msShade", "msTraceShadow", "msResolve", "msOther")) + " ms",
      file=sys.stderr)
