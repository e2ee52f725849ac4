// alpha_caps.cuh — where an alpha-tested triangle is opaque everywhere, and where it is transparent everywhere (device + host code).
//
// The any-hit test of a candidate (k_alpha) draws one rnd() in [0, 1 - 2^-23] and accepts a closest-hit candidate when
// rnd <= opacity, a shadow candidate when rnd < opacity.  A candidate whose opacity is exactly 1 therefore always passes:
// in a closest-hit walk nothing behind it can be drawn for or returned, and in a shadow walk it ends the query when its
// material has transmission <= 0.01 (k_alpha<true> then returns 0 without looking further).  Such a candidate is a CAP.
// The walks still keep a cap as a candidate (it consumes its draw like any other), but they may lower their culling bound
// to its t: nodes and triangles behind it are no longer visited, and the hits, draws and results stay the same bit for bit.
//
// A candidate whose opacity is exactly 0 is a HOLE: a shadow candidate never passes (rnd < 0 is impossible) and a closest-hit one
// passes only when its draw is exactly 0 (the top 23 bits of the pcg output zero), which the seed alone decides.  Its only other
// effect is one pcg step of the seed.  The walks tag every kept cap and hole (traverse.cuh kCandCap / kCandHole); a walk whose kept
// candidates are all caps or holes runs the any-hit loop itself at write-out, from the seed alone, and the path skips k_alpha.
//
// Both are known per micro-triangle of a fixed subdivision level, in the micro-triangle order of omm.cuh (ommBary2Index),
// baked at scene build from the alpha record (device_scene.cuh AlphaRec) by k_cap_bake:
//   capRef[slot]  one word per triangle slot of a tree: kCapNone (neither caps nor holes), kCapAll (every micro-triangle is a cap),
//                 kHoleAll (every micro-triangle is a hole), else the word offset of the triangle's map in capBits: 4^kCapLevel cap
//                 bits, then 4^kCapLevel hole bits (bit i of each = micro-triangle i)
// The closest-hit tree and the shadow rays' non-opaque tree have a reference array each; the shadow one has no caps for materials
// with transmission > 0.01 (their holes stay).  Scenes with opacity micromaps use neither (the micromap lookup decides those walks).
#pragma once
#include "omm.cuh"
#include "vec.cuh"
#include <cstdint>

namespace pt {

// level 5: 1024 micro-triangles, 2 x 128 B of bits per triangle whose micro-triangles are not all of one kind (DESIGN.md §2)
constexpr uint32_t kCapLevel = 5;
constexpr uint32_t kCapMicro = 1u << (2 * kCapLevel);
constexpr uint32_t kCapWords = kCapMicro / 32;
constexpr uint32_t kCapNone = 0xFFFFFFFFu, kCapAll = 0xFFFFFFFEu, kHoleAll = 0xFFFFFFFDu;
// what a micro-triangle is (capState)
enum : int
{
  kMicroOther = 0,
  kMicroCap = 1,
  kMicroHole = 2,
};
// a micro-triangle whose texel footprint is wider than this along an axis is not baked (it is not a cap); SynthSponza's foliage at
// level 5 spans 16 x 16 texels of its 2048^2 atlas
constexpr int kCapMaxFootprint = 64;

// is the micro-triangle under (u, v) (traversal-order barycentrics with the mirrored-instance swap undone) a cap, a hole or neither?
// (ref != kCapNone)
template <typename LoadWord>
PT_HD int capState(uint32_t ref, float u, float v, LoadWord loadWord)
{
  if(ref >= kHoleAll)
    return ref == kCapAll ? kMicroCap : kMicroHole;
  const uint32_t idx = ommBary2Index(u, v, kCapLevel), w = ref + (idx >> 5), b = idx & 31u;
  if((loadWord(w) >> b) & 1u)
    return kMicroCap;
  return ((loadWord(w + kCapWords) >> b) & 1u) ? kMicroHole : kMicroOther;
}

// Cell k of the 2 * 4^level grid cells of a level: lower triangle (iu, iv) or upper triangle (iu, iv) (k >= 4^level) of the
// barycentric grid with n = 2^level steps; false for the cells outside the triangle.  (u, v) of the three corners are returned.
PT_HD bool capCell(uint32_t k, uint32_t level, float cu[3], float cv[3])
{
  const uint32_t n = 1u << level, up = k >> (2 * level), iu = k & (n - 1u), iv = (k >> level) & (n - 1u);
  if(iu + iv + up > n - 1u)
    return false;
  const float s = 1.0f / (float)n;
  if(!up)
  {
    cu[0] = iu * s, cv[0] = iv * s, cu[1] = (iu + 1) * s, cv[1] = iv * s, cu[2] = iu * s, cv[2] = (iv + 1) * s;
  }
  else
  {
    cu[0] = (iu + 1) * s, cv[0] = iv * s, cu[1] = iu * s, cv[1] = (iv + 1) * s, cu[2] = (iu + 1) * s, cv[2] = (iv + 1) * s;
  }
  return true;
}

// Does every texel the sampler can touch for a point of the micro-triangle with corners (cu, cv) pass `passes(alpha byte)`?
// Conservative: the micro-triangle is widened by 1e-5 in barycentric space (the fp32 rounding of ommBary2Index and of the hit's
// barycentrics), its uv hull by the fp32 rounding of the interpolation, and every texel of that box (nearest: the texel under it,
// linear: the 2x2 footprint, through the record's wrap modes) must pass; false for a footprint wider than kCapMaxFootprint.
// alpha8(x, y): alpha byte of level-0 texel (x, y) (wrapped); wrap(i, n, mode): the sampler's wrap of coordinate i.
#pragma nv_exec_check_disable
template <typename Alpha8, typename Wrap, typename Passes>
PT_HD bool footprintPasses(const float uvRec[6], int w0, int h0, uint32_t wrapBits, bool linear, const float cu[3], const float cv[3], Alpha8 alpha8,
                           Wrap wrap, Passes passes)
{
  constexpr float kBaryPad = 1e-5f;
  const int       size[2] = {w0, h0};
  int             lo[2], hi[2];
  for(int a = 0; a < 2; a++)
  {
    const float t0 = uvRec[a], t1 = uvRec[2 + a], t2 = uvRec[4 + a];
    float       mn = 3.0e38f, mx = -3.0e38f;
    for(int c = 0; c < 3; c++)
    {
      const float t = t0 * (1.0f - cu[c] - cv[c]) + t1 * cu[c] + t2 * cv[c];
      mn = fminf(mn, t);
      mx = fmaxf(mx, t);
    }
    const float pad = kBaryPad * (fabsf(t1 - t0) + fabsf(t2 - t0)) + 1e-6f * (fabsf(t0) + fabsf(t1) + fabsf(t2)) + 1e-30f;
    float       x0 = (mn - pad) * (float)size[a], x1 = (mx + pad) * (float)size[a];
    if(!(fabsf(x0) < 1.0e6f && fabsf(x1) < 1.0e6f))
      return false;  // (also NaN)
    const float px = 1e-5f * (fabsf(x0) + fabsf(x1) + 1.0f);
    x0 -= px;
    x1 += px;
    if(linear)
    {
      lo[a] = (int)floorf(x0 - 0.5f);
      hi[a] = (int)floorf(x1 - 0.5f) + 1;
    }
    else
    {
      lo[a] = (int)floorf(x0);
      hi[a] = (int)floorf(x1);
    }
    if(hi[a] - lo[a] >= kCapMaxFootprint)
      return false;
  }
  const int wrapS = (int)(wrapBits & 0xffffu), wrapT = (int)(wrapBits >> 16);
  for(int y = lo[1]; y <= hi[1]; y++)
  {
    const int ty = wrap(y, h0, wrapT);
    for(int x = lo[0]; x <= hi[0]; x++)
      if(!passes(alpha8(wrap(x, w0, wrapS), ty)))
        return false;
  }
  return true;
}

// Is the opacity opacityFromRecord / getOpacity (shade.cuh) computes exactly 1 at every point of the micro-triangle with corners
// (cu, cv)?  Every texel of its footprint (footprintPasses) must pass:
//   MASK   factor x min texel alpha x min vertex-colour alpha >= cutoff with a relative margin of 1e-4 (filtering, products and the
//          barycentric sum round in fp32; every texel of the footprint is at least the minimum, so the filtered value is too)
//   BLEND  the value must be exactly 1: factor 1, no vertex colours, and no texture or nearest filtering of texels of alpha 255
//   OPAQUE (non-opaque only through transmission) opacity is 1 by definition
#pragma nv_exec_check_disable
template <typename Alpha8, typename Wrap>
PT_HD bool capMicroTriangle(const float uvRec[6], int w0, int h0, uint32_t wrapBits, float factor, float cutoff, uint32_t modeFlags, uint32_t colA,
                            bool hasTexture, const float cu[3], const float cv[3], Alpha8 alpha8, Wrap wrap)
{
  const uint32_t mode = modeFlags & 3u;
  if(mode == 0u)
    return true;
  const bool vertexColours = (modeFlags & 8u) != 0, linear = (modeFlags & 4u) != 0;
  if(mode == 2u && (factor != 1.0f || vertexColours || (hasTexture && linear)))
    return false;
  // the texels' alpha bytes that pass, monotone in the byte: every texel of the footprint must pass
  float vcMin = 1.0f;
  if(vertexColours)
  {
    const float m = fminf(fminf((float)(colA & 0xffu), (float)((colA >> 8) & 0xffu)), (float)((colA >> 16) & 0xffu));
    vcMin = m / 255.0f;
  }
  auto passes = [&](int b) { return mode == 2u ? b == 255 : (vcMin > 0.0f && factor * ((float)b / 255.0f) * vcMin >= fmaxf(cutoff, 0.0f) * (1.0f + 1e-4f) + 1e-6f); };
  if(hasTexture && !footprintPasses(uvRec, w0, h0, wrapBits, linear, cu, cv, alpha8, wrap, passes))
    return false;
  return passes(255);
}

// Is that opacity exactly 0 at every point of the micro-triangle (a hole)?  Same footprint as capMicroTriangle:
//   MASK   factor x max texel alpha x max vertex-colour alpha < cutoff with the same relative margin (so a cutoff <= 0 has no holes)
//   BLEND  the value must be exactly 0: factor 0, or every vertex alpha 0, or every texel of the footprint of alpha byte 0 (a
//          filtered sum of zeros is zero)
//   OPAQUE never a hole
#pragma nv_exec_check_disable
template <typename Alpha8, typename Wrap>
PT_HD bool holeMicroTriangle(const float uvRec[6], int w0, int h0, uint32_t wrapBits, float factor, float cutoff, uint32_t modeFlags, uint32_t colA,
                             bool hasTexture, const float cu[3], const float cv[3], Alpha8 alpha8, Wrap wrap)
{
  const uint32_t mode = modeFlags & 3u;
  if(mode == 0u || !(factor >= 0.0f))
    return false;
  const bool vertexColours = (modeFlags & 8u) != 0, linear = (modeFlags & 4u) != 0;
  float      vcMax = 1.0f;
  if(vertexColours)
  {
    const float m = fmaxf(fmaxf((float)(colA & 0xffu), (float)((colA >> 8) & 0xffu)), (float)((colA >> 16) & 0xffu));
    vcMax = m / 255.0f;
  }
  if(mode == 2u)
  {
    if(factor == 0.0f || vcMax == 0.0f)
      return true;
    return hasTexture && footprintPasses(uvRec, w0, h0, wrapBits, linear, cu, cv, alpha8, wrap, [](int b) { return b == 0; });
  }
  auto passes = [&](int b) { return factor * ((float)b / 255.0f) * vcMax < cutoff * (1.0f - 1e-4f) - 1e-6f; };
  if(hasTexture)
    return footprintPasses(uvRec, w0, h0, wrapBits, linear, cu, cv, alpha8, wrap, passes);
  return passes(255);
}

// One cell of k_cap_bake (and of the host check tools/host_caps_check.cpp): false for a cell outside the triangle, else true with the
// micro-triangle's index in `idx` and whether it is a cap and whether it is a hole.
#pragma nv_exec_check_disable
template <typename Alpha8, typename Wrap>
PT_HD bool capBakeCell(uint32_t k, const float uvRec[6], int w0, int h0, uint32_t wrapBits, float factor, float cutoff, uint32_t modeFlags, uint32_t colA,
                       bool hasTexture, Alpha8 alpha8, Wrap wrap, uint32_t& idx, bool& cap, bool& hole)
{
  float cu[3], cv[3];
  if(!capCell(k, kCapLevel, cu, cv))
    return false;
  cap = capMicroTriangle(uvRec, w0, h0, wrapBits, factor, cutoff, modeFlags, colA, hasTexture, cu, cv, alpha8, wrap);
  hole = !cap && holeMicroTriangle(uvRec, w0, h0, wrapBits, factor, cutoff, modeFlags, colA, hasTexture, cu, cv, alpha8, wrap);
  idx = ommBary2Index((cu[0] + cu[1] + cu[2]) / 3.0f, (cv[0] + cv[1] + cv[2]) / 3.0f, kCapLevel);
  return true;
}

}  // namespace pt
