// dlss_guides.cuh — arithmetic of the path tracer's DLSS variant (guide images for DLSS Ray Reconstruction).
//
// Reference: shaders/dlss_util.h (EnvBRDFApprox2, calculateMotionVector) as the DLSS variant of processPixel calls them
// (shaders/gltf_pathtrace.slang:240-263, 628-651), and the storage formats of the six guide images (src/dlss.cpp:59-66).
// fp32 operations in the shader's order; Slang's floatNxN(...) constructors fill rows, so mul(M, v) is row r of M dotted
// with v.  The conversions to binary16 (round to nearest even) and UNORM8 (round(clamp(x, 0, 1) * 255), ties away from
// zero) are the driver's image stores in the reference -- unpinned; the oracle uses the same rules (DESIGN.md section 4).
// Compiled for the host through tools/host_shim.h by tests/test_dlss_guides.py.
#pragma once
#include <cuda_fp16.h>

#include "vec.cuh"

namespace pt {

// Specular albedo for DLSS (Ray Tracing Gems, chapter 32 fit): EnvBRDFApprox2(SpecularColor, alpha, NoV)
PT_HD float3 dlssEnvBRDFApprox2(float3 spec, float alpha, float NoV)
{
  NoV = fabsf(NoV);
  const float X0 = 1.0f, X1 = NoV, X2 = NoV * NoV, X3 = NoV * X2;
  const float Y0 = 1.0f, Y1 = alpha, Y2 = alpha * alpha, Y3 = alpha * Y2;
  // mul(M1, X.xy), M1 = (0.99044, -1.28514; 1.29678, -0.755907)
  const float m1x = 0.99044f * X0 + -1.28514f * X1, m1y = 1.29678f * X0 + -0.755907f * X1;
  // mul(M2, X.xyw)
  const float m2x = (1.0f * X0 + 2.92338f * X1) + 59.4188f * X3;
  const float m2y = (20.3225f * X0 + -27.0302f * X1) + 222.592f * X3;
  const float m2z = (121.563f * X0 + 626.13f * X1) + 316.627f * X3;
  // mul(M3, X.xy), M3 = (0.0365463, 3.32707; 9.0632, -9.04756)
  const float m3x = 0.0365463f * X0 + 3.32707f * X1, m3y = 9.0632f * X0 + -9.04756f * X1;
  // mul(M4, X.xzw)
  const float m4x = (1.0f * X0 + 3.59685f * X2) + -1.36772f * X3;
  const float m4y = (9.04401f * X0 + -16.3174f * X2) + 9.22949f * X3;
  const float m4z = (5.56589f * X0 + 19.7886f * X2) + -20.2123f * X3;
  float       bias = (m1x * Y0 + m1y * Y1) * (1.0f / ((m2x * Y0 + m2y * Y1) + m2z * Y3));
  const float scale = (m3x * Y0 + m3y * Y1) * (1.0f / ((m4x * Y0 + m4y * Y1) + m4z * Y3));
  bias *= saturatef(spec.y * 50.0f);  // the reference's hack for a specular reflectance of 0
  const float s = fmaxf(0.0f, scale), b = fmaxf(0.0f, bias);
  return f3(spec.x * s + b, spec.y * s + b, spec.z * s + b);
}

// calculateMotionVector, path-tracer overload: homogeneous current / previous positions (w = 1 surface, w = 0 a point at
// infinity along the view direction) through the current and previous view-projection (glm bytes, mul(v, M)); pixel-space
// (prevNDC - currNDC) * 0.5 * resolution
PT_HD float2 dlssMotionVector(float4 currWorld, float4 prevWorld, const float* prevMVP, const float* currMVP, float2 resolution)
{
  const float4 cc = mul_vM(currWorld, *reinterpret_cast<const Mat4*>(currMVP));
  const float4 pc = mul_vM(prevWorld, *reinterpret_cast<const Mat4*>(prevMVP));
  const float  cx = cc.x / cc.w, cy = cc.y / cc.w;
  const float  px = pc.x / pc.w, py = pc.y / pc.w;
  return f2((px - cx) * 0.5f * resolution.x, (py - cy) * 0.5f * resolution.y);
}

// fp32 -> IEEE binary16 bits, round to nearest even
PT_HD uint16_t dlssHalfBits(float x)
{
  const __half_raw r = __float2half_rn(x);
  return r.x;
}
// fp32 -> UNORM8
PT_HD uint32_t dlssUnorm8(float x) { return (uint32_t)roundf(saturatef(x) * 255.0f); }

// The six guide planes of one pixel, in the reference's formats (src/dlss.cpp:61-66): 28 bytes
struct DlssGuidePixel
{
  uint32_t albedo;           // RGBA8 UNORM
  uint16_t specAlbedo[4];    // RGBA16F
  uint16_t normalRough[4];   // RGBA16F
  uint16_t motion[2];        // RG16F
  uint16_t depth;            // R16F
  uint16_t specHitDist;      // R16F
};

// processPixel's DLSS stores (gltf_pathtrace.slang:632-650) from what the sample carried: the guide albedo (binary16 values),
// normal / roughness (binary16 values), the first-hit position and its previous-frame position, and the specular albedo and hit
// distance as binary16 bits (x: r | g << 16, y: b | distance << 16).  hasSolidHit (radiance.w > 0) gives the
// albedo's alpha, the w of both positions and the NDC depth (1 = far).
PT_HD DlssGuidePixel dlssPackGuides(float3 albedo, float4 normalRough, uint2 specBits, float3 hitPos, float3 hitPosPrev, bool hasSolidHit,
                                    const float* viewProj, const float* prevMVP, float2 imageSize)
{
  DlssGuidePixel g;
  g.albedo = dlssUnorm8(albedo.x) | (dlssUnorm8(albedo.y) << 8) | (dlssUnorm8(albedo.z) << 16) | (dlssUnorm8(hasSolidHit ? 1.0f : 0.0f) << 24);
  g.specAlbedo[0] = (uint16_t)(specBits.x & 0xffffu);
  g.specAlbedo[1] = (uint16_t)(specBits.x >> 16);
  g.specAlbedo[2] = (uint16_t)(specBits.y & 0xffffu);
  g.specAlbedo[3] = dlssHalfBits(1.0f);
  g.normalRough[0] = dlssHalfBits(normalRough.x);
  g.normalRough[1] = dlssHalfBits(normalRough.y);
  g.normalRough[2] = dlssHalfBits(normalRough.z);
  g.normalRough[3] = dlssHalfBits(normalRough.w);
  const float  w = hasSolidHit ? 1.0f : 0.0f;
  const float2 mv = dlssMotionVector(f4(hitPos, w), f4(hitPosPrev, w), prevMVP, viewProj, imageSize);
  g.motion[0] = dlssHalfBits(mv.x);
  g.motion[1] = dlssHalfBits(mv.y);
  float ndcDepth = 1.0f;
  if(hasSolidHit)
  {
    const float4 clip = mul_vM(f4(hitPos, 1.0f), *reinterpret_cast<const Mat4*>(viewProj));
    ndcDepth = clip.z / clip.w;
  }
  g.depth = dlssHalfBits(ndcDepth);
  g.specHitDist = (uint16_t)(specBits.y >> 16);
  return g;
}

}  // namespace pt
