// device_scene.cuh — HBM-resident scene + per-frame parameter blocks shared by all kernels.
//
// Data contract = what SceneVk / MaterialCache / HdrIbl give the reference shaders
// (shaders/gltf_scene_io.h.slang:41-322; shaders/shaderio.h:148-196), re-laid for CUDA:
//   GltfRenderNode[] / GltfShadeMaterial[] / GltfTextureInfo[] / GltfLight[]  : same bytes, AoS
//   GltfRenderPrimitive (7 device addresses)                                  : DevPrim
//   bindless Sampler2D allTextures[]                                          : DevTex[] (tiled mip chains in global memory)
//   HDR env Sampler2D + StructuredBuffer<EnvAccel>                            : float4[] + uint2[]
//   TLAS/BLAS                                                                 : BvhView (+ triMeta)
#pragma once
#include <cuda_runtime.h>

#include "../../include/b200pt.h"
#include "traverse.cuh"

namespace pt {

struct DevPrim
{
  const uint32_t* idx;
  const float*    pos;
  const float*    nrm;
  const uint32_t* col;
  const float*    tan;
  const float*    uv0;
  const float*    uv1;
};

struct DevTex
{
  // RGBA8 mip pyramid in plain global memory, every level stored as 4x4-texel tiles (64 B: a bilinear footprint
  // mostly stays inside one tile).  Filtering happens in fp32 in the kernel, so the texture unit would only ever
  // point-sample -- and with one texture object per lane every TEX became a waterfall loop over the distinct
  // handles in the warp (SASS: R2UR + BRA.U.ANY around each of the 24 fetches of a shaded hit).
  const uchar4*   texels;
  const uint32_t* levelOfs;  // texel offset of every level from `texels`
  int             w0, h0;
  float           maxLevel;
  int             wrapS, wrapT;  // glTF enums
  int             srgb;
  int             magLinear, minLinear, mipLinear;
};

// Everything the stochastic alpha test of ONE non-opaque triangle needs (getOpacity, pathtrace_functions.h.slang:189-260),
// gathered at scene build: 64 B = four 128-bit loads, against the nine dependent gathers of the generic path (candidate ->
// triMeta -> render node -> primitive -> indices -> uv -> material -> texture info -> texture descriptor) that made the
// any-hit kernels latency-bound (long-scoreboard stalls).
struct AlphaRec
{
  float         uv[6];        // the three vertices' texture coordinates of the set the alpha texture reads ((0,0) if absent)
  const uchar4* lv0;          // level-0 texels of the base-colour / diffuse texture (tiled), nullptr = no texture (alpha 1)
  int           w0, h0;
  uint32_t      wrap;         // wrapS | wrapT << 16 (glTF enums)
  float         factor;       // pbrBaseColorFactor.a (pbrDiffuseFactor.a for specular-glossiness)
  float         cutoff;
  uint32_t      modeFlags;    // bits 0-1 alphaMode, bit 2 magnification filter is linear, bit 3 vertex colours present
  uint32_t      colA;         // vertex colour alphas: a0 | a1 << 8 | a2 << 16 (UNORM8)
  float         transmission; // material.transmissionFactor (<= 0.01: a passing candidate blocks the shadow ray)
};
static_assert(sizeof(AlphaRec) == 64, "AlphaRec is four 16-byte loads");

// The vertex attributes of ONE triangle of a render primitive, gathered at scene build (object space, shared by all
// instances of the primitive): twelve 128-bit loads instead of the dependent chain index -> 3 vertices x {position, normal,
// uv0, uv1, colour, tangent} of narrow loads that getHitState (get_hit.h.slang:59-173) otherwise walks.
struct ShadeRec
{
  // twelve float4, laid out so that every attribute is read by named components (no address arithmetic on the device):
  //   v[0] = pos0.xyz | flags      v[1] = pos1.xyz | col0     v[2] = pos2.xyz | col1     v[3] = nrm0.xyz | col2
  //   v[4] = nrm1.xyz | uv0[0].x   v[5] = nrm2.xyz | uv0[0].y v[6] = uv0[1].xy, uv0[2].xy
  //   v[7] = uv1[0].xy, uv1[1].xy  v[8] = uv1[2].xy | 0 | 0   v[9..11] = tangent 0..2 (xyzw)
  // flags: bit 0 normals, 1 uv0, 2 uv1, 3 colours, 4 tangents present (else the reference's fallbacks apply)
  float4 v[12];
};
static_assert(sizeof(ShadeRec) == 192, "ShadeRec is twelve 16-byte loads");

// ---- per-triangle derivations from a render node's material, shared by b200pt_set_scene (host) and the scene-edit kernels ----

// material index of a render node (-1 = material 0)
PT_HD uint32_t materialOf(const b200pt_render_node& node) { return node.materialID > 0 ? (uint32_t)node.materialID : 0u; }

// the instance flags of a material's triangles (getInstanceFlag, src/gltf_scene_rtx.cpp:271-295)
PT_HD uint32_t triFlags(const b200pt_shade_material& m)
{
  uint32_t flags = 0;
  if(m.transmissionFactor == 0.0f && m.alphaMode == 0 && m.diffuseTransmissionFactor == 0.0f)
    flags |= TRI_OPAQUE;
  if(m.doubleSided == 1 || m.thicknessFactor > 0.0f || m.transmissionFactor > 0.0f)
    flags |= TRI_NOCULL;
  return flags;
}

// The alpha-test record of one non-opaque triangle with vertex indices i0..i2 of a primitive (uv0 / uv1 / colors may be null).
// `textures` are the DevTex records and level0(t) the level-0 texels of texture t (the host keeps them in its own table, the
// device reads them through the record's level offsets).
#pragma nv_exec_check_disable
template <class Level0>
PT_HD AlphaRec alphaRecOf(const b200pt_shade_material& m, const b200pt_texture_info* texInfos, const DevTex* textures, uint32_t numTextures,
                          Level0 level0, const float* uv0, const float* uv1, const uint32_t* colors, uint32_t i0, uint32_t i1, uint32_t i2)
{
  AlphaRec r{};
  r.modeFlags = (uint32_t)m.alphaMode & 3u;
  r.cutoff = m.alphaCutoff;
  r.transmission = m.transmissionFactor;
  const bool     specGloss = m.pbrModel == 1;
  const uint16_t slot = specGloss ? m.pbrDiffuseTexture : m.pbrBaseColorTexture;
  r.factor = specGloss ? m.pbrDiffuseFactor[3] : m.pbrBaseColorFactor[3];
  if(slot > 0)
  {
    const b200pt_texture_info& ti = texInfos[slot];
    const float*               uv = ti.texCoord ? uv1 : uv0;
    if(uv)
    {
      const uint32_t vi[3] = {i0, i1, i2};
      for(int c = 0; c < 3; c++)
      {
        r.uv[c * 2] = uv[vi[c] * 2];
        r.uv[c * 2 + 1] = uv[vi[c] * 2 + 1];
      }
    }
    if(ti.index >= 0 && (uint32_t)ti.index < numTextures)
    {
      const DevTex& dt = textures[ti.index];
      r.lv0 = level0(ti.index);
      r.w0 = dt.w0;
      r.h0 = dt.h0;
      r.wrap = ((uint32_t)dt.wrapS & 0xffffu) | ((uint32_t)dt.wrapT << 16);
      if(dt.magLinear)
        r.modeFlags |= 4u;
    }
  }
  if(colors)
  {
    r.modeFlags |= 8u;
    r.colA = (colors[i0] >> 24) | ((colors[i1] >> 24) << 8) | ((colors[i2] >> 24) << 16);
  }
  return r;
}

struct DevScene
{
  const b200pt_render_node*    nodes;
  const DevPrim*               prims;
  const b200pt_shade_material* mats;
  const b200pt_texture_info*   texInfos;
  const DevTex*                textures;
  const b200pt_light*          lights;
  int                          numLights;
  int                          numTextures;
  BvhView                      bvh;       // closest-hit walks: ONE tree over every triangle; TRI_OPAQUE per triangle decides hit vs candidate
  BvhView                      bvhO;      // shadow walks, phase 0: FORCE_OPAQUE triangles only (any hit ends the query)
  BvhView                      bvhA;      // shadow walks, phase 1: non-opaque triangles only (candidates); shares bvhO's triangle array
  int                          hasAlpha;  // the scene has non-opaque triangles (the any-hit kernels are launched)
  const uint2*                 triMeta;   // per triangle slot of `bvh`: (rnode | flags<<28, primitiveID)
  const uint2*                 triMetaS;  // per triangle slot of bvhO / bvhA (== triMeta in scenes without non-opaque triangles)
  const uint32_t*              matOfSlot; // per triangle slot of `bvh`: material index (key of the material-sorted shade queue)
  int                          numMaterials;
  const ShadeRec*              shadeRecs; // one per triangle of every render primitive
  const uint32_t*              shadeIdx;  // per triangle slot of `bvh`: index into shadeRecs
  const AlphaRec*              alphaRecs; // one per non-opaque triangle, in bvhA's leaf order
  const uint32_t*              alphaIdx;  // per triangle slot of `bvh`: index into alphaRecs (0xFFFFFFFF for opaque triangles)
  uint32_t                     alphaBaseS; // first non-opaque slot of the split triangle array: record = slot - alphaBaseS
  const float4*                envRgba;  // lat-long radiance, pdf in .w
  const uint2*                 envAccel; // (alias, q bits)
  const float*                 lutSrgb;  // 512 floats: sRGB decode table, then i/255 (staged into shared memory per block)
  int                          envW, envH;
};

// the fields of b200pt_frame_info in which the views of one b200pt_render_views call may differ
struct ViewPose
{
  float viewMatrix[16], viewInv[16], viewProjMatrix[16], prevMVP[16];
};

struct FrameParams
{
  b200pt_frame_info    fi;
  b200pt_push_constant pc;
  int                  width, height;
  int                  tileY0, tileRows;
  int                  bandRows, bandWorld, bandRank;  // interleaved tiles: bandWorld > 1 (then tileY0 == 0)
  uint32_t             numPaths;  // path slots of this launch chain = pixels * batch
  // Frame batching (b200pt_set_frame_batch): `batch` consecutive frames of a static camera run as ONE wavefront.  Slot i
  // belongs to pixel i % pixels of frame pc.frameCount + i / pixels; pc holds the FIRST frame's constants, frame b adds b to
  // frameCount and b * numSamples to totalSamples (what the host loop would have passed, src/renderer_pathtracer.cpp:1496-1574).
  uint32_t             pixels;    // tileRows * width
  int                  batch;     // >= 1
  // Views (b200pt_render_views): `views` camera poses of ONE frame run as one wavefront.  Slot i belongs to pixel i % pixels of
  // view i / pixels; every view shares the frame's constants except its pose, poses[v].  At most one of batch and views is above 1.
  int                  views;     // >= 1
  const ViewPose*      poses;     // views > 1: one per view, on the device
  // DLSS frames: objectToWorld of every render node as the previous frame saw it (16 floats each, glm order), or null when no
  // transform changed since that frame (pushConst.prevRenderNodeObjectToWorld, src/renderer_pathtracer.cpp:1553-1561)
  const float*         prevObjectToWorld;
};

// the camera of a path slot: its view's pose, or F.fi's with one view
struct Camera
{
  const float *viewMatrix, *viewInv, *viewProjMatrix, *prevMVP;
};

PT_D uint32_t pixelOf(const FrameParams& F, uint32_t i) { return F.batch > 1 || F.views > 1 ? i % F.pixels : i; }
PT_D uint32_t frameOf(const FrameParams& F, uint32_t i) { return F.batch > 1 ? i / F.pixels : 0u; }
PT_D Camera   cameraOf(const FrameParams& F, uint32_t i)
{
  if(F.views > 1)
  {
    const ViewPose& v = F.poses[i / F.pixels];
    return {v.viewMatrix, v.viewInv, v.viewProjMatrix, v.prevMVP};
  }
  return {F.fi.viewMatrix, F.fi.viewInv, F.fi.viewProjMatrix, F.fi.prevMVP};
}
// the slot renders the first frame of an accumulation (its sample overwrites the image, frame-0 outputs are written)
PT_D bool isFirstFrame(const FrameParams& F, uint32_t i) { return (F.pc.flags & B200PT_PT_FIRST_FRAME) != 0 && (F.batch <= 1 || i < F.pixels); }

// global pixel row of tile pixel p (seeds always use global coordinates)
PT_D uint32_t pixelRow(const FrameParams& F, uint32_t p)
{
  const uint32_t l = p / (uint32_t)F.width;
  if(F.bandWorld <= 1)
    return (uint32_t)F.tileY0 + l;
  return ((l / (uint32_t)F.bandRows) * (uint32_t)F.bandWorld + (uint32_t)F.bandRank) * (uint32_t)F.bandRows + l % (uint32_t)F.bandRows;
}

// ---- wavefront path state (SoA, one slot per pixel of the tile) --------------------------------
// 16-byte records so every access is one 128-bit load/store.
struct PathState
{
  float4*   rayO;    // origin.xyz | cone width
  float4*   rayD;    // direction.xyz | tmax
  float4*   hit;     // t | u | v | triangle slot (bits; 0xFFFFFFFF = miss)
  float4*   thr;     // throughput.xyz | lastSamplePdf
  float4*   rad;     // radiance.xyz | scatterBounces (bits)
  float4*   misc;    // maxRoughness.xy | flags (bits) | seed (bits)
  uint4*    medium;  // fp16x3 extinction | fp16x3 scatter | fp16 anisotropy (packed) | sample index
  float4*   pixSum;  // per-pixel sum of the frame's samples (rgb + solid flag)
  float4*   shO;     // shadow ray origin.xyz | tmax
  float4*   shD;     // shadow ray direction.xyz | unused
  float4*   shC;     // NEE contribution.xyz | unused
  float4*   firstHit;  // first frame only: world position of the sample's first surface hit | 1 (primary miss: direction | 0)
  // any-hit candidates of the ray last traced for the path (closest-hit ray, then the shadow ray): up to kCand
  // nearest non-opaque hits as t | u | v | triangle slot, written by the traversal kernels and consumed by the
  // dense alpha / resolve kernels
  float4*   cand[kCand];
  uint2*    candInfo;  // x: count (bit 31: an opaque occluder ended the shadow query) | y: global id of the last candidate
  // denoiser guides of the sample's first hit (GuideScratch, pathtrace_functions.h.slang:79-88; null unless b200pt_set_guide_outputs):
  // albedo.xyz | roughness and normal.xyz | 1 (0: the primary ray missed), every value rounded through fp16 like the reference's float16_t fields
  float4*   guideA;
  float4*   guideN;
  // DLSS scratch of the sample's first hit (null unless b200pt_set_dlss_guides): its previous-frame world position | 1 (primary
  // miss: direction | 0), and GuideScratch's specular albedo + specular hit distance as binary16 bits (r | g << 16, b | dist << 16)
  float4*   prevHit;
  uint2*    dlssSpec;
};

// a DLSS frame (never batched) on a handle whose pools carry the DLSS scratch
PT_D bool isDlssFrame(const PathState& P, const FrameParams& F) { return P.dlssSpec != nullptr && (F.pc.flags & B200PT_PT_USE_DLSS) != 0; }

// flags word in misc.z
enum : uint32_t
{
  PF_DEPTH_MASK = 0xffffu,
  PF_INSIDE = 1u << 16,
  PF_SOLID = 1u << 17,
  PF_POST_VOLUME = 1u << 18,   // post stage runs the in-volume RR rule instead of the surface one
  PF_SHADOW_VALID = 1u << 19,
  PF_SHADOW_INSIDE = 1u << 20, // TraceShadow(initialInside = true)
  PF_CATCHER = 1u << 21,       // the path sits on the shadow-catcher plane: the post stage runs handleShadowCatcher's second half
  PF_SPEC_CAPTURE = 1u << 22,  // DLSS: GuideScratch::captureSpecularHit, the next Trace records the specular hit distance
};

struct Queues
{
  uint32_t* qTrace;   // paths to trace + shade this iteration
  uint32_t* qPost;    // paths entering the shadow / RR stage
  uint32_t* qNext;    // paths for the next iteration
  uint32_t* counters; // [0] = count(qTrace) [1] = count(qPost) [2] = count(qNext)
};

struct DevStats
{
  unsigned long long closestRays, shadowRays, shadedHits, pathsStarted, nodesVisited, trisTested;
  unsigned long long warpIters, busyLaneIters;  // counter build only: traversal-loop iterations per warp, busy lanes summed
  unsigned long long errorFlags;                // bit 0: a traversal stack overflowed (the walk was incomplete)
};

}  // namespace pt
