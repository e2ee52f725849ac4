"""The count behind the alpha caps' subdivision level (csrc/alpha_caps.cuh kCapLevel, DESIGN.md §2): for SynthSponza (bench.py's
scene), the share of micro-triangles of its alpha-MASK foliage that are opaque everywhere at levels 3-6 -- the share of candidate hits
that land on a cap, the hits being spread evenly over the leaf quads -- and the bytes of bits per mapped triangle.  CPU only.

    python scripts/alpha_cap_levels.py [--levels 3 4 5 6]
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--levels", type=int, nargs="+", default=[3, 4, 5, 6])
    a = ap.parse_args()
    from vk_gltf_renderer_b200 import omm, synth
    scn = synth.synth_sponza(seed=1234)
    for level in a.levels:
        st = omm.bake_opacity_micromaps(scn, level=level)
        print(f"level {level}: {st['triangles']} foliage triangles, opaque micro-triangles {100.0 * st['opaque'] / st['micro']:.1f} %, "
              f"{4 ** level // 8} B of bits per mapped triangle")


if __name__ == "__main__":
    main()
