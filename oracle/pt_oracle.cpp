// =================================================================================================
// pt_oracle.cpp — CPU ORACLE for the vk_gltf_renderer path tracer.   *** TEST INFRASTRUCTURE ***
//
// Scalar fp32 restatement of the reference hot path, used ONLY as the checker by tests/,
// __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.  The product
// (vk_gltf_renderer_b200/csrc, libb200pt.so) never links, imports or calls anything here.
//
// Restates (reference file:line, relative to /root/reference):
//   processPixel / samplePixel / pathTrace / pathTraceOneBounce     shaders/gltf_pathtrace.slang:87-630
//   sampleLights / sampleEnvironment / MIS / volume / RR / getRay   shaders/pathtrace_functions.h.slang
//   RayQueryRaytracer::Trace / TraceShadow                          shaders/raytracer_interface.h.slang:69-187
//   getHitState                                                     shaders/get_hit.h.slang:44-173
//   evaluateMaterial / getTexture                                   shaders/gltf_material_eval.h.slang:76-457
//   getOpacity / getShadowTransmission                              shaders/pathtrace_functions.h.slang:189-343
//   instance flags (opaque / cull-disable)                          src/gltf_scene_rtx.cpp:271-295
//   DLSS variant: jitter, captures, guide images                    shaders/gltf_pathtrace.slang:135-143, 216-263, 370-377, 564-651,
//                                                                   shaders/pathtrace_functions.h.slang:65-102, 942-988
//   EnvBRDFApprox2 / calculateMotionVector                          shaders/dlss_util.h
// and, in bsdf.h, the EXTERNAL nvpro_core2/nvshaders arithmetic (BSDF, RNG, env sampling ...).
//
// PARITY UNPINNED.  The reference cannot be built or run here (needs Vulkan-RT, slangc,
// nvpro_core2@main — SURVEY.md §8c) and its tests hold no golden vector for this path, so this
// oracle is checked only against analytic known-answer tests (tests/test_oracle_*.py: furnace,
// single-triangle hits, alias-table normalisation, MIS weights, BSDF energy/reciprocity ...).
//
// Hardware any-hit order is unspecified in the reference (raytracer_interface.h.slang:53;
// gltf_pathtrace.slang:798-801).  This oracle — and the CUDA path — pin it as follows:
//   Trace:       closest FORCE_OPAQUE hit first; then the non-opaque candidates nearer than it, strictly
//                front-to-back in (t, global triangle id) order, each consuming one rand(); the first
//                accepted candidate commits, otherwise the opaque hit does.
//   TraceShadow: any FORCE_OPAQUE occluder => 0 without consuming rand(); otherwise all non-opaque
//                candidates front-to-back as in the RayQuery loop (:149-179).
// Both are orders the reference's RayQuery/any-hit semantics allow; they make the result (and the
// RNG stream) independent of the acceleration-structure layout.
// =================================================================================================
#include <algorithm>
#include <atomic>
#include <cfloat>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <thread>
#include <vector>

#include "../include/b200pt.h"
#include "bsdf.h"

using namespace orc;

namespace {

// -------------------------------------------------------------------------------------------------
// scene storage
// -------------------------------------------------------------------------------------------------
struct Prim
{
  std::vector<uint32_t> idx;
  std::vector<float>    pos, nrm, tan, uv0, uv1;
  std::vector<uint32_t> col;
  uint32_t              ntri = 0, nvert = 0;
};

struct MipLevel
{
  int                w, h;
  std::vector<float> rgba;  // linear float, 4 per texel
};
struct Texture
{
  std::vector<MipLevel> mips;
  int                   wrapS, wrapT, magFilter, minFilter, srgb;
};

struct FlatTri  // world-space triangle used by traversal
{
  float3   v0, e1, e2;
  uint32_t rnode;
  uint32_t prim;   // triangle index inside the render primitive
  uint32_t flags;  // bit0 opaque, bit1 cull disabled, bit2 winding flipped (mirrored instance)
};
enum
{
  TRI_OPAQUE = 1,
  TRI_NOCULL = 2,
  TRI_FLIPPED = 4
};

struct BvhNode
{
  float3   lo, hi;
  uint32_t left, right;  // children (inner)
  uint32_t first, count; // leaf range into triOrder (count > 0 => leaf)
};

// per-thread counters, merged into the shared totals when a worker finishes (no atomics per ray)
struct LocalStats
{
  uint64_t closestRays = 0, shadowRays = 0, shadedHits = 0, paths = 0, nodes = 0, tris = 0;
};
static thread_local LocalStats tls;
static thread_local bool        dbgPixel = false;  // reference analogue: doDebug at pushConst.mouseCoord (gltf_pathtrace.slang:553-557)
struct Stats
{
  std::atomic<uint64_t> closestRays{0}, shadowRays{0}, shadedHits{0}, paths{0}, nodes{0}, tris{0};
  void                  merge()
  {
    closestRays += tls.closestRays;
    shadowRays += tls.shadowRays;
    shadedHits += tls.shadedHits;
    paths += tls.paths;
    nodes += tls.nodes;
    tris += tls.tris;
    tls = LocalStats();
  }
};

struct Oracle
{
  std::vector<b200pt_render_node>    nodes;
  std::vector<uint8_t>               visible;
  std::vector<Prim>                  prims;
  std::vector<b200pt_shade_material> mats;
  std::vector<b200pt_texture_info>   texInfos;
  std::vector<Texture>               textures;
  std::vector<b200pt_light>          lights;
  std::vector<FlatTri>               tris;
  struct Tree
  {
    std::vector<uint32_t> triOrder;
    std::vector<BvhNode>  bvh;
  };
  Tree treeOpaque, treeAlpha;  // FORCE_OPAQUE triangles / any-hit (non-opaque) triangles
  // opacity micromaps (src/gltf_scene_omm.cpp: the asset's EXT_mesh_opacity_micromap arrays), keyed by render primitive
  struct Micromap
  {
    std::vector<uint8_t>                  data;
    std::vector<b200pt_micromap_triangle> tris;
  };
  struct PrimOmm
  {
    uint32_t             micromap = 0, base = 0;
    bool                 hasIdx = false;
    std::vector<int32_t> idx;
  };
  std::vector<Micromap> micromaps;
  std::vector<PrimOmm>  primOmm;      // one per linked primitive
  std::vector<int>      ommOfPrim;    // renderPrimID -> primOmm index, -1 = none (sized lazily)
  // environment
  int                   envW = 0, envH = 0;
  std::vector<float>    envRgba;
  std::vector<uint32_t> envAlias;
  std::vector<float>    envQ;
  float                 envIntegral = 0.f;
  Stats                 stats;
};

// -------------------------------------------------------------------------------------------------
// sRGB + texture sampling (Vulkan-style: wrap, bilinear, trilinear, explicit-gradient LOD)
// -------------------------------------------------------------------------------------------------
static float srgbToLinear(float c)
{
  return (c <= 0.04045f) ? c / 12.92f : powf((c + 0.055f) / 1.055f, 2.4f);
}
static float linearToSrgb(float c)
{
  return (c <= 0.0031308f) ? c * 12.92f : 1.055f * powf(c, 1.0f / 2.4f) - 0.055f;
}

static void buildTexture(Texture& T, const b200pt_texture& src)
{
  T.wrapS = src.wrapS;
  T.wrapT = src.wrapT;
  T.magFilter = src.magFilter;
  T.minFilter = src.minFilter;
  T.srgb = src.srgb;
  // level 0 as 8-bit, then successive 2x box/linear downsampling re-quantised to 8 bit per level
  // (reference: vkCmdBlitImage chain with VK_FILTER_LINEAR on the UNORM/SRGB image,
  //  src/gltf_scene_vk.cpp:1254-1332: each level is an 8-bit image again)
  int                  w = src.width, h = src.height;
  std::vector<uint8_t> cur(src.rgba8, src.rgba8 + (size_t)w * h * 4);
  float                lutL[256], lutS[256];  // 8-bit decode tables (same values as the per-texel formulas)
  for(int i = 0; i < 256; i++)
  {
    lutL[i] = (float)i / 255.0f;
    lutS[i] = srgbToLinear((float)i / 255.0f);
  }
  for(;;)
  {
    MipLevel L;
    L.w = w;
    L.h = h;
    L.rgba.resize((size_t)w * h * 4);
    for(size_t i = 0; i < (size_t)w * h; i++)
    {
      for(int c = 0; c < 4; c++)
        L.rgba[i * 4 + c] = (T.srgb && c < 3) ? lutS[cur[i * 4 + c]] : lutL[cur[i * 4 + c]];
    }
    T.mips.push_back(std::move(L));
    if(w == 1 && h == 1)
      break;
    int                  nw = std::max(1, w / 2), nh = std::max(1, h / 2);
    std::vector<uint8_t> nxt((size_t)nw * nh * 4);
    const MipLevel&      P = T.mips.back();
    for(int y = 0; y < nh; y++)
      for(int x = 0; x < nw; x++)
      {
        // linear-filter blit: sample the source at the destination texel centre
        float sx = (x + 0.5f) * (float)w / (float)nw - 0.5f;
        float sy = (y + 0.5f) * (float)h / (float)nh - 0.5f;
        int   x0 = (int)floorf(sx), y0 = (int)floorf(sy);
        float fx = sx - x0, fy = sy - y0;
        int   x1 = std::min(x0 + 1, w - 1), y1 = std::min(y0 + 1, h - 1);
        x0 = std::max(x0, 0);
        y0 = std::max(y0, 0);
        for(int c = 0; c < 4; c++)
        {
          float a = P.rgba[((size_t)y0 * w + x0) * 4 + c], b = P.rgba[((size_t)y0 * w + x1) * 4 + c];
          float cc = P.rgba[((size_t)y1 * w + x0) * 4 + c], d = P.rgba[((size_t)y1 * w + x1) * 4 + c];
          float v = (a * (1 - fx) + b * fx) * (1 - fy) + (cc * (1 - fx) + d * fx) * fy;
          if(T.srgb && c < 3)
            v = linearToSrgb(v);
          nxt[((size_t)y * nw + x) * 4 + c] = (uint8_t)std::min(255.0f, std::max(0.0f, floorf(v * 255.0f + 0.5f)));
        }
      }
    cur.swap(nxt);
    w = nw;
    h = nh;
  }
}

static int wrapCoord(int i, int n, int mode)
{
  if(mode == 33071)  // CLAMP_TO_EDGE
    return std::min(std::max(i, 0), n - 1);
  if(mode == 33648)  // MIRRORED_REPEAT
  {
    int p = 2 * n;
    int m = ((i % p) + p) % p;
    return m < n ? m : p - 1 - m;
  }
  return ((i % n) + n) % n;  // REPEAT
}

static float4 fetchTexel(const Texture& T, const MipLevel& L, int x, int y)
{
  x = wrapCoord(x, L.w, T.wrapS);
  y = wrapCoord(y, L.h, T.wrapT);
  const float* p = &L.rgba[((size_t)y * L.w + x) * 4];
  return f4(p[0], p[1], p[2], p[3]);
}

static float4 sampleLevel(const Texture& T, int level, float2 uv, bool linear)
{
  const MipLevel& L = T.mips[level];
  float           x = uv.x * (float)L.w, y = uv.y * (float)L.h;
  if(!linear)
    return fetchTexel(T, L, (int)floorf(x), (int)floorf(y));
  x -= 0.5f;
  y -= 0.5f;
  float  fx0 = floorf(x), fy0 = floorf(y);
  float  fx = x - fx0, fy = y - fy0;
  int    x0 = (int)fx0, y0 = (int)fy0;
  float4 a = fetchTexel(T, L, x0, y0), b = fetchTexel(T, L, x0 + 1, y0);
  float4 c = fetchTexel(T, L, x0, y0 + 1), d = fetchTexel(T, L, x0 + 1, y0 + 1);
  float4 top = a * (1.0f - fx) + b * fx;
  float4 bot = c * (1.0f - fx) + d * fx;
  return top * (1.0f - fy) + bot * fy;
}

// lambda = log2(max(|ddx * size|, |ddy * size|)); lambda <= 0 -> magnification (level 0).
// Sampler quirks kept from the reference: the mip mode follows magFilter, and magFilter goes through the same table
// as minFilter, so 9984 / 9986 there are NEAREST too (gltf_scene_vk.cpp:922-942).
static float4 sampleTexture(const Texture& T, float2 uv, float2 ddx, float2 ddy, bool useGrad)
{
  const bool magLinear = !(T.magFilter == 9728 || T.magFilter == 9984 || T.magFilter == 9986);
  const bool minLinear = !(T.minFilter == 9728 || T.minFilter == 9984 || T.minFilter == 9986);
  const bool mipLinear = magLinear;
  if(!useGrad)
    return sampleLevel(T, 0, uv, magLinear);
  const float w = (float)T.mips[0].w, h = (float)T.mips[0].h;
  const float lx = sqrtf(ddx.x * w * ddx.x * w + ddx.y * h * ddx.y * h);
  const float ly = sqrtf(ddy.x * w * ddy.x * w + ddy.y * h * ddy.y * h);
  const float rho = fmaxf(lx, ly);
  float       lambda = log2f(rho);
  const float maxLevel = (float)(T.mips.size() - 1);
  if(!(lambda > 0.0f))
    return sampleLevel(T, 0, uv, magLinear);
  lambda = fminf(lambda, maxLevel);
  if(!mipLinear)
  {
    int lv = (int)fminf(maxLevel, fmaxf(0.0f, ceilf(lambda + 0.5f) - 1.0f));
    return sampleLevel(T, lv, uv, minLinear);
  }
  int   l0 = (int)floorf(lambda);
  int   l1 = std::min(l0 + 1, (int)maxLevel);
  float f = lambda - (float)l0;
  float4 a = sampleLevel(T, l0, uv, minLinear);
  if(f == 0.0f || l1 == l0)
    return a;
  float4 b = sampleLevel(T, l1, uv, minLinear);
  return a * (1.0f - f) + b * f;
}

// -------------------------------------------------------------------------------------------------
// environment: alias table + pdf in alpha (nvvk::HdrIbl, external; call site src/renderer.cpp:1994)
// -------------------------------------------------------------------------------------------------
static float buildAliasmap(const std::vector<float>& data, std::vector<uint32_t>& alias, std::vector<float>& q)
{
  const uint32_t size = (uint32_t)data.size();
  float          sum = 0.f;
  for(float d : data)
    sum += d;
  const float average = sum / (float)size;
  alias.resize(size);
  q.resize(size);
  for(uint32_t i = 0; i < size; i++)
  {
    q[i] = data[i] / average;
    alias[i] = i;
  }
  std::vector<uint32_t> part(size);
  uint32_t              s = 0u, large = size;
  for(uint32_t i = 0; i < size; ++i)
  {
    if(q[i] < 1.f)
      part[s++] = i;
    else
      part[--large] = i;
  }
  for(s = 0; s < large && large < size; ++s)
  {
    const uint32_t j = part[s], k = part[large];
    alias[j] = k;
    const float diff = 1.f - q[j];
    q[k] -= diff;
    if(q[k] < 1.0f)
      large++;
  }
  return sum;
}

static void setEnvironment(Oracle& o, const float* rgb, int w, int h)
{
  o.envW = w;
  o.envH = h;
  o.envRgba.resize((size_t)w * h * 4);
  std::vector<float> importance((size_t)w * h);
  const float        stepPhi = M_TWO_PI_F / (float)w;
  const float        stepTheta = M_PI_F / (float)h;
  for(int y = 0; y < h; y++)
  {
    const float theta0 = (float)y * stepTheta;
    const float theta1 = (float)(y + 1) * stepTheta;
    const float area = (cosf(theta0) - cosf(theta1)) * stepPhi;
    for(int x = 0; x < w; x++)
    {
      size_t i = (size_t)y * w + x;
      float  r = rgb[i * 3], g = rgb[i * 3 + 1], b = rgb[i * 3 + 2];
      o.envRgba[i * 4] = r;
      o.envRgba[i * 4 + 1] = g;
      o.envRgba[i * 4 + 2] = b;
      importance[i] = area * fmaxf(r, fmaxf(g, b));
    }
  }
  o.envIntegral = buildAliasmap(importance, o.envAlias, o.envQ);
  const float inv = 1.0f / o.envIntegral;
  for(size_t i = 0; i < (size_t)w * h; i++)
    o.envRgba[i * 4 + 3] = fmaxf(o.envRgba[i * 4], fmaxf(o.envRgba[i * 4 + 1], o.envRgba[i * 4 + 2])) * inv;
}

// HDR lat-long lookup: linear filter, level 0, repeat in u, clamp in v
static float4 sampleEnvTex(const Oracle& o, float2 uv)
{
  const int w = o.envW, h = o.envH;
  float     x = uv.x * (float)w - 0.5f, y = uv.y * (float)h - 0.5f;
  float     fx0 = floorf(x), fy0 = floorf(y);
  float     fx = x - fx0, fy = y - fy0;
  int       x0 = (int)fx0, y0 = (int)fy0;
  auto      at = [&](int xi, int yi) {
    xi = ((xi % w) + w) % w;
    yi = std::min(std::max(yi, 0), h - 1);
    const float* p = &o.envRgba[((size_t)yi * w + xi) * 4];
    return f4(p[0], p[1], p[2], p[3]);
  };
  float4 a = at(x0, y0), b = at(x0 + 1, y0), c = at(x0, y0 + 1), d = at(x0 + 1, y0 + 1);
  float4 top = a * (1.0f - fx) + b * fx;
  float4 bot = c * (1.0f - fx) + d * fx;
  return top * (1.0f - fy) + bot * fy;
}

// nvshaders/hdr_env_sampling: alias pick + uniform direction inside the texel
static float4 environmentSample(const Oracle& o, float3 xi, float3& toLight)
{
  const uint32_t width = (uint32_t)o.envW, height = (uint32_t)o.envH;
  const uint32_t size = width * height;
  const uint32_t idx = std::min((uint32_t)(xi.x * (float)size), size - 1);
  uint32_t       envIdx;
  float          xi_y = xi.y;
  if(xi_y < o.envQ[idx])
  {
    envIdx = idx;
    xi_y /= o.envQ[idx];
  }
  else
  {
    envIdx = o.envAlias[idx];
    xi_y = (xi_y - o.envQ[idx]) / (1.0f - o.envQ[idx]);
  }
  const uint32_t py = envIdx / width;
  const uint32_t px = envIdx % width;
  const float    u = ((float)px + xi_y) / (float)width;
  const float    phi = u * M_TWO_PI_F - M_PI_F;
  const float    sinPhi = sinf(phi), cosPhi = cosf(phi);
  const float    stepTheta = M_PI_F / (float)height;
  const float    theta0 = (float)py * stepTheta;
  const float    cosTheta = cosf(theta0) * (1.0f - xi.z) + cosf(theta0 + stepTheta) * xi.z;
  const float    theta = acosf(cosTheta);
  const float    sinTheta = sinf(theta);
  const float    v = theta * M_1_PI_F;
  toLight = f3(cosPhi * sinTheta, cosTheta, sinPhi * sinTheta);
  return sampleEnvTex(o, f2(u, v));
}

// -------------------------------------------------------------------------------------------------
// BVH2 (SAH, binned) over flattened world-space triangles
// -------------------------------------------------------------------------------------------------
static void triBounds(const FlatTri& t, float3& lo, float3& hi)
{
  float3 v1 = t.v0 + t.e1, v2 = t.v0 + t.e2;
  lo = vmin(t.v0, vmin(v1, v2));
  hi = vmax(t.v0, vmax(v1, v2));
  // pad by a few ulp: v0+e1 is a rounded reconstruction of the vertex
  float3 pad = vmax(f3(fabsf(lo.x), fabsf(lo.y), fabsf(lo.z)), f3(fabsf(hi.x), fabsf(hi.y), fabsf(hi.z))) * 4e-7f + f3(1e-30f);
  lo = lo - pad;
  hi = hi + pad;
}

static float halfArea(float3 lo, float3 hi)
{
  float3 d = hi - lo;
  return d.x * d.y + d.y * d.z + d.z * d.x;
}

static void buildBvh(const Oracle& scene, Oracle::Tree& o, const std::vector<uint32_t>& ids)
{
  const uint32_t n = (uint32_t)ids.size();
  o.triOrder = ids;
  o.bvh.clear();
  if(n == 0)
    return;
  const uint32_t      nAll = (uint32_t)scene.tris.size();
  std::vector<float3> lo(nAll), hi(nAll), ce(nAll);
  for(uint32_t k = 0; k < n; k++)
  {
    const uint32_t i = ids[k];
    triBounds(scene.tris[i], lo[i], hi[i]);
    ce[i] = (lo[i] + hi[i]) * 0.5f;
  }
  o.bvh.reserve(2 * n);
  struct Job
  {
    uint32_t node, first, count;
  };
  std::vector<Job> stack;
  o.bvh.push_back({});
  stack.push_back({0, 0, n});
  while(!stack.empty())
  {
    Job j = stack.back();
    stack.pop_back();
    float3 blo = f3(FLT_MAX), bhi = f3(-FLT_MAX), clo = f3(FLT_MAX), chi = f3(-FLT_MAX);
    for(uint32_t i = j.first; i < j.first + j.count; i++)
    {
      uint32_t t = o.triOrder[i];
      blo = vmin(blo, lo[t]);
      bhi = vmax(bhi, hi[t]);
      clo = vmin(clo, ce[t]);
      chi = vmax(chi, ce[t]);
    }
    BvhNode& N = o.bvh[j.node];
    N.lo = blo;
    N.hi = bhi;
    N.left = N.right = 0;
    N.first = j.first;
    N.count = j.count;
    if(j.count <= 4)
      continue;
    // binned SAH
    const int NB = 16;
    float     bestCost = FLT_MAX;
    int       bestAxis = -1, bestBin = -1;
    float3    ext = chi - clo;
    for(int ax = 0; ax < 3; ax++)
    {
      float e = (&ext.x)[ax];
      if(e <= 0.f)
        continue;
      float3   binLo[NB], binHi[NB];
      uint32_t binCnt[NB];
      for(int b = 0; b < NB; b++)
      {
        binLo[b] = f3(FLT_MAX);
        binHi[b] = f3(-FLT_MAX);
        binCnt[b] = 0;
      }
      float scale = (float)NB / e, c0 = (&clo.x)[ax];
      for(uint32_t i = j.first; i < j.first + j.count; i++)
      {
        uint32_t t = o.triOrder[i];
        int      b = std::min(NB - 1, (int)(((&ce[t].x)[ax] - c0) * scale));
        binCnt[b]++;
        binLo[b] = vmin(binLo[b], lo[t]);
        binHi[b] = vmax(binHi[b], hi[t]);
      }
      float    rightArea[NB];
      uint32_t rightCnt[NB];
      float3   rl = f3(FLT_MAX), rh = f3(-FLT_MAX);
      uint32_t rc = 0;
      for(int b = NB - 1; b > 0; b--)
      {
        rl = vmin(rl, binLo[b]);
        rh = vmax(rh, binHi[b]);
        rc += binCnt[b];
        rightArea[b] = rc ? halfArea(rl, rh) : 0.f;
        rightCnt[b] = rc;
      }
      float3   ll = f3(FLT_MAX), lh = f3(-FLT_MAX);
      uint32_t lc = 0;
      for(int b = 0; b < NB - 1; b++)
      {
        ll = vmin(ll, binLo[b]);
        lh = vmax(lh, binHi[b]);
        lc += binCnt[b];
        if(lc == 0 || rightCnt[b + 1] == 0)
          continue;
        float cost = halfArea(ll, lh) * (float)lc + rightArea[b + 1] * (float)rightCnt[b + 1];
        if(cost < bestCost)
        {
          bestCost = cost;
          bestAxis = ax;
          bestBin = b;
        }
      }
    }
    uint32_t mid;
    if(bestAxis < 0)
    {
      mid = j.first + j.count / 2;  // all centroids coincide: split by order
    }
    else
    {
      float e = (&ext.x)[bestAxis], scale = (float)NB / e, c0 = (&clo.x)[bestAxis];
      auto  it = std::partition(o.triOrder.begin() + j.first, o.triOrder.begin() + j.first + j.count, [&](uint32_t t) {
        int b = std::min(NB - 1, (int)(((&ce[t].x)[bestAxis] - c0) * scale));
        return b <= bestBin;
      });
      mid = (uint32_t)(it - o.triOrder.begin());
      if(mid == j.first || mid == j.first + j.count)
        mid = j.first + j.count / 2;
    }
    uint32_t l = (uint32_t)o.bvh.size();
    o.bvh.push_back({});
    o.bvh.push_back({});
    o.bvh[j.node].left = l;
    o.bvh[j.node].right = l + 1;
    o.bvh[j.node].count = 0;
    stack.push_back({l, j.first, mid - j.first});
    stack.push_back({l + 1, mid, j.first + j.count - mid});
  }
}

// -------------------------------------------------------------------------------------------------
// ray / triangle (Moeller-Trumbore with explicit fma chains — the CUDA kernel uses the same
// sequence so (t,u,v) agree bit-for-bit) and the "next hit in (t, id) order" query
// -------------------------------------------------------------------------------------------------
struct Ray
{
  float3 o;
  float  tmin;
  float3 d;
  float  tmax;
};
struct Hit
{
  float    t;
  uint32_t tri;  // index into o.tris
  float    u, v;
};

static inline float3 crossFma(float3 a, float3 b)
{
  return f3(fmaf(a.y, b.z, -(a.z * b.y)), fmaf(a.z, b.x, -(a.x * b.z)), fmaf(a.x, b.y, -(a.y * b.x)));
}
static inline float dotFma(float3 a, float3 b) { return fmaf(a.z, b.z, fmaf(a.y, b.y, a.x * b.x)); }

// returns true and (t,u,v,det) if the ray's supporting line crosses the triangle
static inline bool intersectTri(const FlatTri& T, const Ray& r, float& t, float& u, float& v, float& det)
{
  const float3 pvec = crossFma(r.d, T.e2);
  det = dotFma(T.e1, pvec);
  if(det == 0.0f)
    return false;
  const float  inv = 1.0f / det;
  const float3 tvec = r.o - T.v0;
  u = dotFma(tvec, pvec) * inv;
  if(u < 0.0f || u > 1.0f)
    return false;
  const float3 qvec = crossFma(tvec, T.e1);
  v = dotFma(r.d, qvec) * inv;
  if(v < 0.0f || u + v > 1.0f)
    return false;
  t = dotFma(T.e2, qvec) * inv;
  return true;
}

static inline bool slab(const BvhNode& N, const Ray& r, float3 invD, float tmax, float& tnear)
{
  float t0 = r.tmin, t1 = tmax;
  for(int a = 0; a < 3; a++)
  {
    const float tlo = ((&N.lo.x)[a] - (&r.o.x)[a]) * (&invD.x)[a];
    const float thi = ((&N.hi.x)[a] - (&r.o.x)[a]) * (&invD.x)[a];
    float       tn = fminf(tlo, thi), tf = fmaxf(tlo, thi);  // fminf/fmaxf drop NaNs (0 * inf)
    // widen a few ulp so the box test stays conservative w.r.t. the (inexact) triangle test
    tn = tn - fabsf(tn) * 1e-6f;
    tf = tf + fabsf(tf) * 1e-6f;
    t0 = fmaxf(t0, tn);
    t1 = fminf(t1, tf);
  }
  tnear = t0;
  return t0 <= t1;
}

// -------------------------------------------------------------------------------------------------
// opacity micromaps: what the hardware traversal does with them (docs/RENDERING_ARCHITECTURE.md:65-78,
// raytracer_interface.h.slang:93-100): an OPAQUE micro-triangle is a committed hit without an any-hit
// invocation, a TRANSPARENT one is culled, the UNKNOWN states are any-hit candidates as before.
// Micro-triangle order: VK_EXT_opacity_micromap bary2index (specification text, restated; unpinned).
// -------------------------------------------------------------------------------------------------
enum
{
  OMM_TRANSPARENT = 0,
  OMM_OPAQUE = 1,
  OMM_UNKNOWN = 2
};

static uint32_t ommInterleave(uint32_t x)
{
  uint32_t r = 0;
  for(int b = 0; b < 16; b++)
    r |= ((x >> b) & 1u) << (2 * b);
  return r;
}

static uint32_t ommBary2Index(float u, float v, uint32_t level)
{
  u = std::min(std::max(u, 0.0f), 1.0f);
  v = std::min(std::max(v, 0.0f), 1.0f);
  const uint32_t n = 1u << level;
  const float    fu = u * (float)n, fv = v * (float)n;
  uint32_t       iu = (uint32_t)fu, iv = (uint32_t)fv;
  const float    uf = fu - (float)iu, vf = fv - (float)iv;
  iu = std::min(iu, n - 1u);
  iv = std::min(iv, n - 1u);
  const uint32_t iuv = iu + iv;
  if(iuv >= n)
    iu -= iuv - n + 1u;
  uint32_t iw = ~(iu + iv);
  if(uf + vf >= 1.0f && iuv < n - 1u)
    --iw;
  const uint32_t b0 = ~(iu ^ iw) & (n - 1u);
  const uint32_t t = (iu ^ iv) & b0;
  uint32_t       f = t;
  f ^= f >> 1;
  f ^= f >> 2;
  f ^= f >> 4;
  f ^= f >> 8;
  const uint32_t b1 = ((f ^ iu) & ~b0) | t;
  return ommInterleave(b0) | (ommInterleave(b1) << 1);
}

// state of the micro-triangle of flattened triangle T under barycentrics (u, v) (weights of the primitive's 2nd / 3rd vertex)
static int ommState(const Oracle& o, const FlatTri& T, float u, float v)
{
  if(o.primOmm.empty())
    return OMM_UNKNOWN;
  const uint32_t prim = (uint32_t)o.nodes[T.rnode].renderPrimID;
  const int      k = prim < o.ommOfPrim.size() ? o.ommOfPrim[prim] : -1;
  if(k < 0)
    return OMM_UNKNOWN;
  const Oracle::PrimOmm& po = o.primOmm[(size_t)k];
  const int32_t          idx = po.hasIdx ? po.idx[T.prim] : (int32_t)T.prim;
  if(idx == B200PT_OMM_INDEX_FULLY_TRANSPARENT)
    return OMM_TRANSPARENT;
  if(idx == B200PT_OMM_INDEX_FULLY_OPAQUE)
    return OMM_OPAQUE;
  if(idx < 0)
    return OMM_UNKNOWN;
  const Oracle::Micromap&         M = o.micromaps[po.micromap];
  const b200pt_micromap_triangle& R = M.tris[(size_t)idx + po.base];
  const uint32_t                  m = ommBary2Index(u, v, R.subdivisionLevel);
  if(R.format == B200PT_OMM_FORMAT_4_STATE)
  {
    const uint32_t st = (M.data[R.dataOffset + (m >> 2)] >> ((m & 3u) * 2u)) & 3u;
    return st < 2u ? (int)st : OMM_UNKNOWN;
  }
  return (int)((M.data[R.dataOffset + (m >> 3)] >> (m & 7u)) & 1u);
}

// closest hit with (t,id) strictly greater than (loT, loId) in lexicographic order, t in (tmin,tmax).
// ommWant >= 0: only hits whose micro-triangle state is `ommWant` count (the others are skipped).
// cull: apply back-face culling (closest-hit rays) honouring TRI_NOCULL.
static bool nextHit(const Oracle& scene, const Oracle::Tree& o, const Ray& r, bool cull, float loT, uint32_t loId, bool haveLo, Hit& best, bool anyExit = false,
                    int ommWant = -1)
{
  if(o.bvh.empty())
    return false;
  const float3 invD = f3(1.0f / r.d.x, 1.0f / r.d.y, 1.0f / r.d.z);
  best.t = r.tmax;
  best.tri = 0xFFFFFFFFu;
  uint32_t stack[128];
  int      sp = 0;
  stack[sp++] = 0;
  uint64_t nodes = 0, tris = 0;
  while(sp)
  {
    const BvhNode& N = o.bvh[stack[--sp]];
    float          tn;
    nodes++;
    if(!slab(N, r, invD, best.t, tn))
      continue;
    if(N.count)
    {
      for(uint32_t i = N.first; i < N.first + N.count; i++)
      {
        const uint32_t id = o.triOrder[i];
        const FlatTri& T = scene.tris[id];
        float          t, u, v, det;
        tris++;
        if(!intersectTri(T, r, t, u, v, det))
          continue;
        if(cull && !(T.flags & TRI_NOCULL))
        {
          // front face <=> det > 0 (CCW seen from the ray origin); mirrored instances flip it
          const bool front = (T.flags & TRI_FLIPPED) ? (det < 0.0f) : (det > 0.0f);
          if(!front)
            continue;
        }
        if(!(t > r.tmin && t < r.tmax))
          continue;
        if(haveLo && !(t > loT || (t == loT && id > loId)))
          continue;
        if(ommWant >= 0 && !(t < best.t || (t == best.t && id < best.tri)))
          continue;
        if(ommWant >= 0 && ommState(scene, T, (T.flags & TRI_FLIPPED) ? v : u, (T.flags & TRI_FLIPPED) ? u : v) != ommWant)
          continue;
        if(t < best.t || (t == best.t && id < best.tri))
        {
          best.t = t;
          best.tri = id;
          best.u = u;
          best.v = v;
          if(anyExit)
          {
            sp = 0;
            break;
          }
        }
      }
    }
    else
    {
      // near child first
      const BvhNode& L = o.bvh[N.left];
      const BvhNode& R = o.bvh[N.right];
      float          tl, tr;
      bool           hl = slab(L, r, invD, best.t, tl), hr = slab(R, r, invD, best.t, tr);
      if(hl && hr)
      {
        if(tl <= tr)
        {
          stack[sp++] = N.right;
          stack[sp++] = N.left;
        }
        else
        {
          stack[sp++] = N.left;
          stack[sp++] = N.right;
        }
      }
      else if(hl)
        stack[sp++] = N.left;
      else if(hr)
        stack[sp++] = N.right;
    }
  }
  tls.nodes += nodes;
  tls.tris += tris;
  if(best.tri == 0xFFFFFFFFu)
    return false;
  if(scene.tris[best.tri].flags & TRI_FLIPPED)
    std::swap(best.u, best.v);
  return true;
}

// -------------------------------------------------------------------------------------------------
// vertex access (gltf_vertex_access.h.slang)
// -------------------------------------------------------------------------------------------------
static inline float3 ld3(const std::vector<float>& a, uint32_t i) { return f3(a[i * 3], a[i * 3 + 1], a[i * 3 + 2]); }
static inline float2 ld2(const std::vector<float>& a, uint32_t i) { return f2(a[i * 2], a[i * 2 + 1]); }
static inline float4 ld4(const std::vector<float>& a, uint32_t i) { return f4(a[i * 4], a[i * 4 + 1], a[i * 4 + 2], a[i * 4 + 3]); }
static inline float4 unpackUnorm4x8(uint32_t p)
{
  return f4((float)((p >> 0) & 0xFF) / 255.0f, (float)((p >> 8) & 0xFF) / 255.0f, (float)((p >> 16) & 0xFF) / 255.0f,
            (float)((p >> 24) & 0xFF) / 255.0f);
}
static inline float3 mixBary(float3 a, float3 b, float3 c, float3 bary) { return a * bary.x + b * bary.y + c * bary.z; }
static inline float2 mixBary(float2 a, float2 b, float2 c, float3 bary) { return a * bary.x + b * bary.y + c * bary.z; }

static float2 interpTexCoord(const Prim& P, int channel, const uint32_t tri[3], float3 bary)
{
  const std::vector<float>& uv = channel ? P.uv1 : P.uv0;
  if(uv.empty())
    return f2(0.0f, 0.0f);
  return mixBary(ld2(uv, tri[0]), ld2(uv, tri[1]), ld2(uv, tri[2]), bary);
}
static float4 interpColor(const Prim& P, const uint32_t tri[3], float3 bary)
{
  if(P.col.empty())
    return f4(1, 1, 1, 1);
  return unpackUnorm4x8(P.col[tri[0]]) * bary.x + unpackUnorm4x8(P.col[tri[1]]) * bary.y + unpackUnorm4x8(P.col[tri[2]]) * bary.z;
}

// -------------------------------------------------------------------------------------------------
// getHitState (get_hit.h.slang:59-173)
// -------------------------------------------------------------------------------------------------
struct HitState
{
  float3 pos, nrm;
  float4 color;
  float3 geonrm, shadowPos;
  float2 uv[2];
  float3 tangent, bitangent;
  float  texelDensity;
  bool   frontFace;
};

static HitState getHitState(const Prim& P, float3 bary, const mat4& W2O, const mat4& O2W, uint32_t triangleID, float3 rayDir)
{
  HitState       hit;
  const uint32_t tri[3] = {P.idx[triangleID * 3], P.idx[triangleID * 3 + 1], P.idx[triangleID * 3 + 2]};
  const float3   pos0 = ld3(P.pos, tri[0]), pos1 = ld3(P.pos, tri[1]), pos2 = ld3(P.pos, tri[2]);
  const float3   position = pos0 * bary.x + pos1 * bary.y + pos2 * bary.z;
  hit.pos = xfPoint(O2W, position);

  const float3 geoNormal = normalize(cross(pos1 - pos0, pos2 - pos0));
  hit.geonrm = normalize(xfNormal(W2O, geoNormal));

  float3 nrm0 = geoNormal, nrm1 = geoNormal, nrm2 = geoNormal, normal = geoNormal;
  if(!P.nrm.empty())
  {
    nrm0 = ld3(P.nrm, tri[0]);
    nrm1 = ld3(P.nrm, tri[1]);
    nrm2 = ld3(P.nrm, tri[2]);
    normal = nrm0 * bary.x + nrm1 * bary.y + nrm2 * bary.z;
  }
  hit.nrm = normalize(xfNormal(W2O, normal));

  hit.frontFace = dot(hit.geonrm, rayDir) < 0.0f;
  const float sideFlip = hit.frontFace ? 1.0f : -1.0f;

  float3 shadowPos = pointOffset(position, pos0, pos1, pos2, nrm0 * sideFlip, nrm1 * sideFlip, nrm2 * sideFlip, bary);
  hit.shadowPos = xfPoint(O2W, shadowPos);

  hit.uv[0] = interpTexCoord(P, 0, tri, bary);
  hit.uv[1] = interpTexCoord(P, 1, tri, bary);

  if(!P.uv0.empty())
  {
    const float2 uv0 = ld2(P.uv0, tri[0]), uv1 = ld2(P.uv0, tri[1]), uv2 = ld2(P.uv0, tri[2]);
    const float3 we1 = xfVector(O2W, pos1 - pos0);
    const float3 we2 = xfVector(O2W, pos2 - pos0);
    const float  wArea = length(cross(we1, we2));
    const float2 duv1 = uv1 - uv0, duv2 = uv2 - uv0;
    const float  uvArea = fabsf(duv1.x * duv2.y - duv1.y * duv2.x);
    hit.texelDensity = sqrtf(fmaxf(uvArea, 1e-20f) / fmaxf(wArea, 1e-20f));
  }
  else
    hit.texelDensity = 0.0f;

  hit.color = interpColor(P, tri, bary);

  float4 tng[3];
  if(!P.tan.empty())
  {
    tng[0] = ld4(P.tan, tri[0]);
    tng[1] = ld4(P.tan, tri[1]);
    tng[2] = ld4(P.tan, tri[2]);
  }
  else
  {
    float4 t = makeFastTangent(normal);
    tng[0] = tng[1] = tng[2] = t;
  }
  hit.tangent = normalize(mixBary(xyz(tng[0]), xyz(tng[1]), xyz(tng[2]), bary));
  hit.tangent = xfVector(O2W, hit.tangent);
  hit.tangent = normalize(hit.tangent - hit.nrm * dot(hit.nrm, hit.tangent));
  hit.bitangent = cross(hit.nrm, hit.tangent) * tng[0].w;

  if(!hit.frontFace)
    hit.geonrm = -hit.geonrm;
  if(dot(hit.geonrm, hit.nrm) < 0)
  {
    hit.nrm = -hit.nrm;
    hit.tangent = -hit.tangent;
    hit.bitangent = -hit.bitangent;
  }
  float3 r = reflect(normalize(rayDir), hit.nrm);
  if(dot(r, hit.geonrm) < 0)
    hit.nrm = hit.geonrm;
  return hit;
}

// -------------------------------------------------------------------------------------------------
// material evaluation (gltf_material_eval.h.slang)
// -------------------------------------------------------------------------------------------------
#define MICROFACET_MIN_ROUGHNESS 0.0014142f

static float4 getTexture(const Oracle& o, const b200pt_texture_info& ti, const float2 tc[2], float texGrad)
{
  float2 tt = tc[ti.texCoord];
  // KHR_texture_transform: mul(float3(tt,1), uvTransform).xy with glm mat3x2 columns c0,c1,c2
  const float* m = ti.uvTransform;
  tt = f2(m[0] * tt.x + m[2] * tt.y + m[4], m[1] * tt.x + m[3] * tt.y + m[5]);
  if(ti.index < 0 || ti.index >= (int)o.textures.size())
    return f4(1, 1, 1, 1);
  const Texture& T = o.textures[ti.index];
  if(texGrad > 0.0f)
  {
    float2 ddx = f2(m[0] * texGrad, m[1] * texGrad);
    float2 ddy = f2(m[2] * texGrad, m[3] * texGrad);
    return sampleTexture(T, tt, ddx, ddy, true);
  }
  return sampleTexture(T, tt, f2(0, 0), f2(0, 0), false);
}
static float4 sampleLevel0(const Oracle& o, const b200pt_texture_info& ti, float2 uv)
{
  if(ti.index < 0 || ti.index >= (int)o.textures.size())
    return f4(1, 1, 1, 1);
  return sampleTexture(o.textures[ti.index], uv, f2(0, 0), f2(0, 0), false);
}

static float3 multiToSingleScatterAlbedo(float3 rho)
{
  float3 t = f3(4.09712f) + rho * 4.20863f - sqrtv(f3(9.59217f) + rho * 41.6808f + rho * rho * 17.7126f);
  return f3(1.0f) - t * t;
}

static float3 convertSGToMR(float3 diffuse, float3 specular, float glossiness, float& metallic, float2& roughness)
{
  const float ds = 0.04f;
  float       specI = fmaxf(specular.x, fmaxf(specular.y, specular.z));
  metallic = smoothstep(ds + 0.01f, ds + 0.05f, specI);
  float3 baseColor;
  if(metallic > 0.0f)
    baseColor = specular;
  else
  {
    baseColor = diffuse / (1.0f - ds * (1.0f - metallic));
    baseColor = f3(clampf(baseColor.x, 0, 1), clampf(baseColor.y, 0, 1), clampf(baseColor.z, 0, 1));
  }
  float r = 1.0f - glossiness;
  roughness = f2(r * r, r * r);
  return baseColor;
}

struct MeshState
{
  float3 N, T, B, Ng;
  float2 tc[2];
  bool   isInside;
  float  texGrad;
  float4 baseColorVertexMul;
};

static PbrMaterial evaluateMaterial(const Oracle& o, const b200pt_shade_material& material, const MeshState& state)
{
  PbrMaterial pbrMat = defaultPbrMaterial();
  const auto& TI = o.texInfos;
#define TEX(slot) getTexture(o, TI[material.slot], state.tc, state.texGrad)
  if(material.pbrModel == 1)
  {
    float4 diffuse = f4(material.pbrDiffuseFactor[0], material.pbrDiffuseFactor[1], material.pbrDiffuseFactor[2], material.pbrDiffuseFactor[3])
                     * state.baseColorVertexMul;
    float  glossiness = material.pbrGlossinessFactor;
    float3 specular = f3(material.pbrSpecularFactor[0], material.pbrSpecularFactor[1], material.pbrSpecularFactor[2]);
    if(material.pbrDiffuseTexture > 0)
      diffuse *= TEX(pbrDiffuseTexture);
    if(material.pbrSpecularGlossinessTexture > 0)
    {
      float4 s = TEX(pbrSpecularGlossinessTexture);
      specular *= xyz(s);
      glossiness *= s.w;
    }
    pbrMat.baseColor = convertSGToMR(xyz(diffuse), specular, glossiness, pbrMat.metallic, pbrMat.roughness);
    pbrMat.opacity = diffuse.w;
  }
  else
  {
    float4 baseColor = f4(material.pbrBaseColorFactor[0], material.pbrBaseColorFactor[1], material.pbrBaseColorFactor[2], material.pbrBaseColorFactor[3])
                       * state.baseColorVertexMul;
    if(material.pbrBaseColorTexture > 0)
      baseColor *= TEX(pbrBaseColorTexture);
    pbrMat.baseColor = xyz(baseColor);
    pbrMat.opacity = baseColor.w;
    float roughness = material.pbrRoughnessFactor;
    float metallic = material.pbrMetallicFactor;
    if(material.pbrMetallicRoughnessTexture > 0)
    {
      float4 mr = TEX(pbrMetallicRoughnessTexture);
      roughness *= mr.y;
      metallic *= mr.z;
    }
    roughness = fmaxf(roughness, MICROFACET_MIN_ROUGHNESS);
    pbrMat.roughness = f2(roughness * roughness, roughness * roughness);
    pbrMat.metallic = clampf(metallic, 0.0f, 1.0f);
  }

  pbrMat.occlusion = material.occlusionStrength;
  if(material.occlusionTexture > 0)
  {
    float occ = TEX(occlusionTexture).x;
    pbrMat.occlusion = 1.0f + pbrMat.occlusion * (occ - 1.0f);
  }

  pbrMat.N = state.N;
  pbrMat.T = state.T;
  pbrMat.B = state.B;
  pbrMat.Ng = state.Ng;
  bool needsTangentUpdate = false;
  if(material.normalTexture > 0)
  {
    float3 nv = xyz(TEX(normalTexture));
    nv = nv * 2.0f - f3(1.0f);
    nv = nv * f3(material.normalTextureScale, material.normalTextureScale, 1.0f);
    // mul(normal_vector, float3x3(T,B,N)) = nv.x*T + nv.y*B + nv.z*N
    pbrMat.N = normalize(state.T * nv.x + state.B * nv.y + state.N * nv.z);
    needsTangentUpdate = true;
  }

  pbrMat.emissive = f3(material.emissiveFactor[0], material.emissiveFactor[1], material.emissiveFactor[2]);
  if(material.emissiveTexture > 0)
    pbrMat.emissive *= xyz(TEX(emissiveTexture));
  pbrMat.emissive = vmax(f3(0.0f), pbrMat.emissive);

  pbrMat.attenuationColor = f3(material.attenuationColor[0], material.attenuationColor[1], material.attenuationColor[2]);
  pbrMat.attenuationDistance = material.attenuationDistance;
  pbrMat.thickness = material.thicknessFactor;
  if(material.thicknessTexture > 0)
    pbrMat.thickness *= TEX(thicknessTexture).y;

  pbrMat.specularColor = f3(material.specularColorFactor[0], material.specularColorFactor[1], material.specularColorFactor[2]);
  if(material.specularColorTexture > 0)
    pbrMat.specularColor *= xyz(TEX(specularColorTexture));
  pbrMat.specular = material.specularFactor;
  if(material.specularTexture > 0)
    pbrMat.specular *= TEX(specularTexture).w;

  float ior1 = 1.0f, ior2 = material.ior;
  if(state.isInside && (pbrMat.thickness > 0.0f))
  {
    ior1 = ior2;
    ior2 = 1.0f;
  }
  pbrMat.ior1 = ior1;
  pbrMat.ior2 = ior2;

  pbrMat.transmission = material.transmissionFactor;
  if(material.transmissionTexture > 0)
    pbrMat.transmission *= TEX(transmissionTexture).x;

  if(material.multiscatterColorFactor[0] > 0.0f || material.multiscatterColorFactor[1] > 0.0f || material.multiscatterColorFactor[2] > 0.0f)
  {
    float3 ssa = multiToSingleScatterAlbedo(f3(material.multiscatterColorFactor[0], material.multiscatterColorFactor[1], material.multiscatterColorFactor[2]));
    float3 att = -logv(vmax(pbrMat.attenuationColor, f3(0.001f))) / fmaxf(pbrMat.attenuationDistance, 0.001f);
    pbrMat.scatterCoefficient = att * ssa;
  }
  pbrMat.scatterAnisotropy = material.scatterAnisotropy;

  pbrMat.clearcoat = material.clearcoatFactor;
  pbrMat.clearcoatRoughness = material.clearcoatRoughness;
  pbrMat.Nc = pbrMat.N;
  if(material.clearcoatTexture > 0)
    pbrMat.clearcoat *= TEX(clearcoatTexture).x;
  if(material.clearcoatRoughnessTexture > 0)
    pbrMat.clearcoatRoughness *= TEX(clearcoatRoughnessTexture).y;
  if(material.clearcoatNormalTexture > 0)
  {
    float3 nv = xyz(TEX(clearcoatNormalTexture));
    nv = nv * 2.0f - f3(1.0f);
    pbrMat.Nc = normalize(pbrMat.T * nv.x + pbrMat.B * nv.y + pbrMat.Nc * nv.z);
  }
  pbrMat.clearcoatRoughness = fmaxf(pbrMat.clearcoatRoughness, 0.001f);

  float iridescence = material.iridescenceFactor;
  float iridescenceThickness = material.iridescenceThicknessMaximum;
  pbrMat.iridescenceIor = material.iridescenceIor;
  if(material.iridescenceTexture > 0)
    iridescence *= TEX(iridescenceTexture).x;
  if(material.iridescenceThicknessTexture > 0)
  {
    const float t = TEX(iridescenceThicknessTexture).y;
    iridescenceThickness = lerpf(material.iridescenceThicknessMinimum, material.iridescenceThicknessMaximum, t);
  }
  pbrMat.iridescence = (iridescenceThickness > 0.0f) ? iridescence : 0.0f;
  pbrMat.iridescenceThickness = iridescenceThickness;

  float anisotropyStrength = material.anisotropyStrength;
  if(anisotropyStrength > 0.0f)
  {
    float2 dir = f2(1.0f, 0.0f);
    if(material.anisotropyTexture > 0)
    {
      const float4 at = TEX(anisotropyTexture);
      dir = normalize(f2(at.x * 2.0f - 1.0f, at.y * 2.0f - 1.0f));
      anisotropyStrength *= at.z;
    }
    pbrMat.roughness.x = lerpf(pbrMat.roughness.y, 1.0f, anisotropyStrength * anisotropyStrength);
    const float s = material.anisotropyRotation[0], c = material.anisotropyRotation[1];
    dir = f2(c * dir.x + s * dir.y, c * dir.y - s * dir.x);
    pbrMat.T = pbrMat.T * dir.x + pbrMat.B * dir.y;
    needsTangentUpdate = true;
  }

  if(needsTangentUpdate)
  {
    pbrMat.B = normalize(cross(pbrMat.N, pbrMat.T));
    float bitangentSign = signf(dot(state.B, pbrMat.B));
    pbrMat.B = pbrMat.B * bitangentSign;
    pbrMat.T = normalize(cross(pbrMat.B, pbrMat.N) * bitangentSign);
  }

  pbrMat.sheenColor = f3(material.sheenColorFactor[0], material.sheenColorFactor[1], material.sheenColorFactor[2]);
  if(material.sheenColorTexture > 0)
    pbrMat.sheenColor *= xyz(TEX(sheenColorTexture));
  pbrMat.sheenRoughness = material.sheenRoughnessFactor;
  if(material.sheenRoughnessTexture > 0)
    pbrMat.sheenRoughness *= TEX(sheenRoughnessTexture).w;
  pbrMat.sheenRoughness = fmaxf(MICROFACET_MIN_ROUGHNESS, pbrMat.sheenRoughness);

  pbrMat.dispersion = material.dispersion;

  pbrMat.diffuseTransmissionFactor = material.diffuseTransmissionFactor;
  if(material.diffuseTransmissionTexture > 0)
    pbrMat.diffuseTransmissionFactor *= TEX(diffuseTransmissionTexture).w;
  pbrMat.diffuseTransmissionColor = f3(material.diffuseTransmissionColor[0], material.diffuseTransmissionColor[1], material.diffuseTransmissionColor[2]);
  if(material.diffuseTransmissionColorTexture > 0)
    pbrMat.diffuseTransmissionColor *= xyz(TEX(diffuseTransmissionColorTexture));

  pbrMat.retroreflection = material.retroreflectionFactor;
  if(material.retroreflectionTexture > 0)
    pbrMat.retroreflection *= TEX(retroreflectionTexture).x;
#undef TEX
  return pbrMat;
}

// -------------------------------------------------------------------------------------------------
// getOpacity / getShadowTransmission (pathtrace_functions.h.slang:189-343)
// -------------------------------------------------------------------------------------------------
static float getOpacity(const Oracle& o, const b200pt_render_node& node, const Prim& P, uint32_t triangleID, float3 bary)
{
  const b200pt_shade_material& mat = o.mats[std::max(0, node.materialID)];
  if(mat.alphaMode == 0)
    return 1.0f;
  const uint32_t tri[3] = {P.idx[triangleID * 3], P.idx[triangleID * 3 + 1], P.idx[triangleID * 3 + 2]};
  float          a = 1.0f;
  if(mat.pbrModel == 1)
  {
    a = mat.pbrDiffuseFactor[3];
    if(mat.pbrDiffuseTexture > 0)
    {
      const b200pt_texture_info& ti = o.texInfos[mat.pbrDiffuseTexture];
      a *= sampleLevel0(o, ti, interpTexCoord(P, ti.texCoord, tri, bary)).w;
    }
  }
  else
  {
    a = mat.pbrBaseColorFactor[3];
    if(mat.pbrBaseColorTexture > 0)
    {
      const b200pt_texture_info& ti = o.texInfos[mat.pbrBaseColorTexture];
      a *= sampleLevel0(o, ti, interpTexCoord(P, ti.texCoord, tri, bary)).w;
    }
  }
  a *= interpColor(P, tri, bary).w;
  if(mat.alphaMode == 1)
    return a >= mat.alphaCutoff ? 1.0f : 0.0f;
  return a;
}

static float3 getShadowTransmission(const Oracle& o, const b200pt_render_node& node, const Prim& P, uint32_t triangleID, float3 bary, float hitT, float3 rayDir, bool& isInside)
{
  const b200pt_shade_material& mat = o.mats[std::max(0, node.materialID)];
  const float                  tFactor = mat.transmissionFactor;
  if(tFactor <= 0.01f)
    return f3(0.0f);
  const uint32_t tri[3] = {P.idx[triangleID * 3], P.idx[triangleID * 3 + 1], P.idx[triangleID * 3 + 2]};
  float3         normal;
  {
    const float3 v0 = ld3(P.pos, tri[0]), v1 = ld3(P.pos, tri[1]), v2 = ld3(P.pos, tri[2]);
    normal = normalize(cross(v1 - v0, v2 - v0));
    const mat4& W2O = *(const mat4*)node.worldToObject;
    normal = normalize(xfNormal(W2O, normal));
  }
  const float cosTheta = fabsf(dot(rayDir, normal));
  const float fresnel = schlickFresnel(mat.ior, cosTheta);
  float3      cur = f3(mat.pbrBaseColorFactor[0], mat.pbrBaseColorFactor[1], mat.pbrBaseColorFactor[2]) * tFactor;
  cur *= (1.0f - fresnel);
  if(mat.thicknessFactor > 0.0f)
  {
    if(isInside)
    {
      float3 absCoeff = -logv(vmax(f3(mat.attenuationColor[0], mat.attenuationColor[1], mat.attenuationColor[2]), f3(0.001f)))
                        / fmaxf(mat.attenuationDistance, 0.001f);
      float3 scatterCoeff = absCoeff * multiToSingleScatterAlbedo(f3(mat.multiscatterColorFactor[0], mat.multiscatterColorFactor[1], mat.multiscatterColorFactor[2]));
      float3 extinction = absCoeff + scatterCoeff;
      cur *= expv(extinction * -hitT);
      float maxScatter = maxc(scatterCoeff);
      if(maxScatter > 0.001f)
      {
        float maxExt = maxc(extinction);
        cur *= expf(-(hitT * maxExt));
      }
    }
    isInside = !isInside;
  }
  float att = 1.0f;
  {
    float roughness = mat.pbrRoughnessFactor, metallic = mat.pbrMetallicFactor;
    if(mat.pbrMetallicRoughnessTexture > 0)
    {
      const b200pt_texture_info& ti = o.texInfos[mat.pbrMetallicRoughnessTexture];
      float4                     mr = sampleLevel0(o, ti, interpTexCoord(P, ti.texCoord, tri, bary));
      roughness *= mr.y;
      metallic *= mr.z;
    }
    att *= (1.0f - metallic);
    float roughnessEffect = 1.0f - (roughness * roughness);
    att *= lerpf(0.65f, 1.0f, roughnessEffect);
  }
  return cur * att;
}

// -------------------------------------------------------------------------------------------------
// Trace / TraceShadow (raytracer_interface.h.slang:69-187), front-to-back candidate order
// -------------------------------------------------------------------------------------------------
struct HitPayload
{
  float hitT;
  int   rnodeID, rprimID, primitiveID;
  float bx, by;
};

static void Trace(Oracle& o, const Ray& ray, HitPayload& p, uint32_t& seed)
{
  tls.closestRays++;
  p.hitT = INFINITE_F;
  p.rnodeID = p.rprimID = p.primitiveID = -1;
  p.bx = p.by = 0.f;
  auto commit = [&](const Hit& h) {
    const FlatTri& T = o.tris[h.tri];
    p.hitT = h.t;
    p.rnodeID = (int)T.rnode;
    p.rprimID = o.nodes[T.rnode].renderPrimID;
    p.primitiveID = (int)T.prim;
    p.bx = h.u;
    p.by = h.v;
  };
  // 1. closest FORCE_OPAQUE hit
  Hit  ho;
  bool haveOpaque = nextHit(o, o.treeOpaque, ray, true, 0.f, 0u, false, ho);
  const bool omm = !o.primOmm.empty();
  if(omm && !o.treeAlpha.bvh.empty())
  {
    // 1b. a hit on an OPAQUE micro-triangle of an alpha-tested triangle is committed the same way (no any-hit, no rand())
    // (ties at the same t go to the smaller triangle id, like every other comparison of the walk)
    Ray r1 = ray;
    if(haveOpaque)
      r1.tmax = nextafterf(ho.t, INFINITE_F);
    Hit hm;
    if(nextHit(o, o.treeAlpha, r1, true, 0.f, 0u, false, hm, false, OMM_OPAQUE) && (!haveOpaque || hm.t < ho.t || (hm.t == ho.t && hm.tri < ho.tri)))
    {
      ho = hm;
      haveOpaque = true;
    }
  }
  // 2. non-opaque candidates nearer than it, front to back (stochastic alpha, :104-111); with micromaps only the UNKNOWN ones
  if(!o.treeAlpha.bvh.empty())
  {
    Ray r2 = ray;
    if(haveOpaque)
      r2.tmax = ho.t;
    float    loT = 0.f;
    uint32_t loId = 0;
    bool     haveLo = false;
    for(;;)
    {
      Hit h;
      if(!nextHit(o, o.treeAlpha, r2, true, loT, loId, haveLo, h, false, omm ? OMM_UNKNOWN : -1))
        break;
      const FlatTri&            T = o.tris[h.tri];
      const b200pt_render_node& node = o.nodes[T.rnode];
      const float3              bary = f3(1.0f - h.u - h.v, h.u, h.v);
      const float               opacity = getOpacity(o, node, o.prims[node.renderPrimID], T.prim, bary);
      if(rnd(seed) <= opacity)
      {
        commit(h);
        return;
      }
      loT = h.t;
      loId = h.tri;
      haveLo = true;
    }
  }
  if(haveOpaque)
    commit(ho);
}

static float3 TraceShadow(Oracle& o, const Ray& ray, uint32_t& seed, bool initialInside)
{
  tls.shadowRays++;
  // 1. any opaque occluder
  {
    Hit h;
    if(nextHit(o, o.treeOpaque, ray, false, 0.f, 0u, false, h, true))
      return f3(0.0f);
  }
  float3 total = f3(1.0f);
  if(o.treeAlpha.bvh.empty())
    return total;
  const bool omm = !o.primOmm.empty();
  if(omm)
  {
    // an OPAQUE micro-triangle anywhere on the segment is a committed hit as well (:181-184)
    Hit h;
    if(nextHit(o, o.treeAlpha, ray, false, 0.f, 0u, false, h, true, OMM_OPAQUE))
      return f3(0.0f);
  }
  // 2. every non-opaque candidate, front to back (:149-179)
  bool     isInside = initialInside;
  float    prevHitT = 0.f;
  float    loT = 0.f;
  uint32_t loId = 0;
  bool     haveLo = false;
  for(;;)
  {
    Hit h;
    if(!nextHit(o, o.treeAlpha, ray, false, loT, loId, haveLo, h, false, omm ? OMM_UNKNOWN : -1))
      return total;
    const FlatTri&            T = o.tris[h.tri];
    const b200pt_render_node& node = o.nodes[T.rnode];
    const Prim&               P = o.prims[node.renderPrimID];
    float3                    bary = f3(1.0f - h.u - h.v, h.u, h.v);
    float                     opacity = getOpacity(o, node, P, T.prim, bary);
    float                     r = rnd(seed);
    if(r < opacity)
    {
      float  seg = fmaxf(0.0f, h.t - prevHitT);
      float3 cur = getShadowTransmission(o, node, P, T.prim, bary, seg, ray.d, isInside);
      prevHitT = h.t;
      total *= cur;
      if(maxc(total) <= 0.01f)
        return f3(0.0f);
    }
    loT = h.t;
    loId = h.tri;
    haveLo = true;
  }
}

// -------------------------------------------------------------------------------------------------
// lights (nvshaders/light_contrib.h.slang, external — restated)
// -------------------------------------------------------------------------------------------------
struct LightContrib
{
  float3 incidentVector;
  float  halfAngularSize;
  float3 intensity;
  float  distance;
  float  pdf;
};

static LightContrib singleLightContribution(const b200pt_light& light, float3 surfacePos, float3 surfaceNormal, float2 xi)
{
  (void)surfaceNormal;
  LightContrib c;
  c.incidentVector = f3(0.0f);
  c.halfAngularSize = 0.0f;
  c.intensity = f3(0.0f);
  c.distance = INFINITE_F;
  c.pdf = DIRAC;
  float        irradiance = 0.0f;
  const float3 ldir = f3(light.direction[0], light.direction[1], light.direction[2]);
  if(light.type == 1)
  {
    c.incidentVector = ldir;
    c.halfAngularSize = light.angularSizeOrInvRange * 0.5f;
    irradiance = light.intensity;
  }
  else if(light.type == 2 || light.type == 3)
  {
    float3 l2s = surfacePos - f3(light.position[0], light.position[1], light.position[2]);
    float  distance = sqrtf(dot(l2s, l2s));
    float  rDistance = 1.0f / distance;
    c.distance = distance;
    c.incidentVector = l2s * rDistance;
    float attenuation = 1.0f;
    if(light.angularSizeOrInvRange > 0.0f)
    {
      attenuation = square(saturate(1.0f - square(square(distance * light.angularSizeOrInvRange))));
      if(attenuation == 0.0f)
        return c;
    }
    float spotlight = 1.0f;
    if(light.type == 2)
    {
      float lDotD = dot(c.incidentVector, ldir);
      float directionAngle = acosf(clampf(lDotD, -1.0f, 1.0f));
      spotlight = 1.0f - smoothstep(light.innerAngle, light.outerAngle, directionAngle);
      if(spotlight == 0.0f)
        return c;
    }
    if(light.radius > 0.0f)
    {
      c.halfAngularSize = atanf(fminf(light.radius * rDistance, 1.0f));
      float solidAngleOverPi = square(c.halfAngularSize);
      float radianceTimesPi = light.intensity / square(light.radius);
      irradiance = radianceTimesPi * solidAngleOverPi;
    }
    else
      irradiance = light.intensity * square(rDistance);
    irradiance *= spotlight * attenuation;
  }
  c.intensity = f3(light.color[0], light.color[1], light.color[2]) * irradiance;
  if(c.halfAngularSize > 0.0f)
  {
    // uniform direction inside the cone of half-angle halfAngularSize about -incidentVector
    const float  cosMax = cosf(c.halfAngularSize);
    const float  cosT = 1.0f - xi.x * (1.0f - cosMax);
    const float  sinT = sqrtf(fmaxf(0.0f, 1.0f - cosT * cosT));
    const float  phi = M_TWO_PI_F * xi.y;
    const float3 axis = -c.incidentVector;
    const float4 t4 = makeFastTangent(axis);
    const float3 T = normalize(xyz(t4));
    const float3 B = cross(axis, T);
    const float3 d = normalize(T * (sinT * cosf(phi)) + B * (sinT * sinf(phi)) + axis * cosT);
    c.incidentVector = -d;
    c.pdf = 1.0f / (M_TWO_PI_F * (1.0f - cosMax));
  }
  return c;
}

// -------------------------------------------------------------------------------------------------
// per-frame context + direct lighting (pathtrace_functions.h.slang:357-492)
// -------------------------------------------------------------------------------------------------
struct Ctx
{
  Oracle*                     o;
  const b200pt_frame_info*    fi;
  const b200pt_push_constant* pc;
  bool                        dlss;               // a DLSS frame (pc carries B200PT_PT_USE_DLSS): the USE_DLSS_SHADER captures
  const float*                prevObjectToWorld;  // DLSS: previous-frame objectToWorld per render node (16 floats, glm order), or null: camera-only motion
};

struct DirectLight
{
  float3 direction, radianceOverPdf;
  float  distance, pdf;
};

static void techniqueProbabilities(const Ctx& c, float& lightWeight, float& envWeight)
{
  lightWeight = (c.o->lights.size() > 0) ? 0.5f : 0.0f;
  envWeight = (!(c.fi->flags & B200PT_SCENE_USE_HDR_ENVIRONMENT) || c.fi->envIntensity > 0.0f) ? 0.5f : 0.0f;
  float total = lightWeight + envWeight;
  if(total > 0.0f)
  {
    lightWeight /= total;
    envWeight /= total;
  }
}

static void sampleLights(const Ctx& c, float3 pos, float3 normal, uint32_t& seed, DirectLight& dl, bool isVolumeSample)
{
  float3 radiance = f3(0.0f);
  dl.pdf = 0.0f;
  dl.distance = INFINITE_F;
  dl.radianceOverPdf = f3(0.0f);
  dl.direction = f3(0.0f);
  float envPdf = 0.0f;
  float lightWeight, envWeight;
  techniqueProbabilities(c, lightWeight, envWeight);
  if(lightWeight == 0.0f && envWeight == 0.0f)
    return;
  const bool sampleLight = (rnd(seed) < lightWeight);
  const int  numLights = (int)c.o->lights.size();
  if(sampleLight)
  {
    float               selectionPdf = 1.0f / (float)numLights;
    int                 lightIndex = std::min((int)(rnd(seed) * (float)numLights), numLights - 1);
    const b200pt_light& light = c.o->lights[lightIndex];
    float3              cullNormal = (isVolumeSample && light.type == 1) ? -f3(light.direction[0], light.direction[1], light.direction[2]) : normal;
    float               r1 = rnd(seed), r2 = rnd(seed);
    LightContrib        contrib = singleLightContribution(light, pos, cullNormal, f2(r1, r2));
    dl.direction = -contrib.incidentVector;
    dl.distance = contrib.distance;
    radiance = contrib.intensity / (selectionPdf * lightWeight);
    dl.pdf = (contrib.pdf == DIRAC) ? DIRAC : selectionPdf * contrib.pdf;
  }
  if(envWeight > 0 && dl.pdf != DIRAC)
  {
    // HDR environment only (BASELINE configs run --envSystem 1; the physical sky is out of scope)
    if(!sampleLight)
    {
      float  a = rnd(seed), b = rnd(seed), cc = rnd(seed);
      float4 rp = environmentSample(*c.o, f3(a, b, cc), dl.direction);
      envPdf = rp.w;
      radiance = xyz(rp) * c.fi->envIntensity / (envPdf * envWeight);
      dl.direction = rotate(dl.direction, f3(0, 1, 0), c.fi->envRotation);
    }
    else
    {
      float3 dir = rotate(dl.direction, f3(0, 1, 0), -c.fi->envRotation);
      float4 rp = sampleEnvTex(*c.o, getSphericalUv(dir));
      envPdf = rp.w;
    }
  }
  float misWeight = 1.0f;
  if(dl.pdf != DIRAC)
  {
    float pdfSum = lightWeight * dl.pdf + envWeight * envPdf;
    if(pdfSum > 0.0f)
      misWeight = (sampleLight ? lightWeight * dl.pdf : envWeight * envPdf) / pdfSum;
    dl.pdf = pdfSum;
  }
  radiance *= misWeight;
  dl.radianceOverPdf = radiance;
}

static void sampleEnvironment(const Ctx& c, float3 direction, float3& envColor, float& envPdf)
{
  float3 dir = rotate(direction, f3(0, 1, 0), -c.fi->envRotation);
  float4 env = sampleEnvTex(*c.o, getSphericalUv(dir));
  envColor = xyz(env) * c.fi->envIntensity;
  envPdf = env.w;
}

static float computeEnvHitMisWeight(const Ctx& c, float lastSamplePdf, float envPdf)
{
  // an infinite pdf is a delta as well: a refraction with ior1 == ior2 sends every microfacet normal to the same direction,
  // and the lobe's Jacobian divides by zero.  inf / (inf + x) would be NaN.
  if(lastSamplePdf == DIRAC || std::isinf(lastSamplePdf))
    return 1.0f;
  float lw, ew;
  techniqueProbabilities(c, lw, ew);
  return lastSamplePdf / (lastSamplePdf + ew * envPdf);
}

// -------------------------------------------------------------------------------------------------
// path state + helpers (pathtrace_functions.h.slang)
// -------------------------------------------------------------------------------------------------
static float3 safeOffsetRay(float3 p, float3 dir)
{
  const float scaleValue = 256.0f;
  const int   sx = (int)(scaleValue * dir.x), sy = (int)(scaleValue * dir.y), sz = (int)(scaleValue * dir.z);
  const float3 op = f3(asfloat(asint(p.x) + ((p.x < 0) ? -sx : sx)), asfloat(asint(p.y) + ((p.y < 0) ? -sy : sy)),
                       asfloat(asint(p.z) + ((p.z < 0) ? -sz : sz)));
  const float origin = 1.0f / 32.0f, floatScale = 1.0f / 65536.0f;
  return f3(fabsf(p.x) < origin ? p.x + floatScale * dir.x : op.x, fabsf(p.y) < origin ? p.y + floatScale * dir.y : op.y,
            fabsf(p.z) < origin ? p.z + floatScale * dir.z : op.z);
}

struct VolumeMedium
{
  float3 extinction, scatterCoefficient;  // values already rounded through fp16
  float  scatterAnisotropy;
};
static float3 volumeExtinctionCoefficient(const PbrMaterial& m)
{
  float3 absC = -logv(vmax(m.attenuationColor, f3(0.001f))) / fmaxf(m.attenuationDistance, 0.001f);
  return absC + m.scatterCoefficient;
}
static VolumeMedium makeVolumeMedium(const PbrMaterial& m)
{
  VolumeMedium v;
  v.extinction = roundHalf(volumeExtinctionCoefficient(m));
  v.scatterCoefficient = roundHalf(m.scatterCoefficient);
  v.scatterAnisotropy = roundHalf(m.scatterAnisotropy);
  return v;
}
static bool hasVolumeMedium(const VolumeMedium& v) { return maxc(v.extinction) > 0.0f || maxc(v.scatterCoefficient) > 0.0f; }

// value of x after a round trip through IEEE binary16 (round to nearest even): the reference's float16_t guide fields
static inline float half16(float x) { return (float)(_Float16)x; }

static inline uint16_t halfBits(float x)
{
  const _Float16 h = (_Float16)x;
  uint16_t       b;
  memcpy(&b, &h, 2);
  return b;
}
static uint32_t unorm8(float x) { return (uint32_t)roundf(fminf(fmaxf(x, 0.0f), 1.0f) * 255.0f); }

// ---- DLSS guide arithmetic (shaders/dlss_util.h), restated: Slang matrices are row-major, mul(M, v)[r] = dot(row r, v), dot and
//      mul sum left to right, rcp(x) = 1 / x, mad(a, b, c) = a * b + c (unfused, like the rest of the oracle)
template <int N>
static float dotN(const float* a, const float* b)
{
  float r = a[0] * b[0];
  for(int k = 1; k < N; k++)
    r = r + a[k] * b[k];
  return r;
}
template <int N>
static void mulMv(const float (&M)[N][N], const float* v, float* out)
{
  for(int r = 0; r < N; r++)
    out[r] = dotN<N>(M[r], v);
}

// EnvBRDFApprox2(SpecularColor, alpha, NoV): Ray Tracing Gems chapter 32 fit of the split-sum specular albedo
static float3 envBRDFApprox2(float3 specularColor, float alpha, float NoV)
{
  NoV = fabsf(NoV);
  const float X[4] = {1.0f, NoV, NoV * NoV, NoV * (NoV * NoV)};
  const float Y[4] = {1.0f, alpha, alpha * alpha, alpha * (alpha * alpha)};
  static const float M1[2][2] = {{0.99044f, -1.28514f}, {1.29678f, -0.755907f}};
  static const float M2[3][3] = {{1.f, 2.92338f, 59.4188f}, {20.3225f, -27.0302f, 222.592f}, {121.563f, 626.13f, 316.627f}};
  static const float M3[2][2] = {{0.0365463f, (float)3.32707}, {9.0632f, (float)-9.04756}};
  static const float M4[3][3] = {{1.f, 3.59685f, -1.36772f}, {9.04401f, -16.3174f, 9.22949f}, {5.56589f, 19.7886f, -20.2123f}};
  const float xy[2] = {X[0], X[1]}, xyw[3] = {X[0], X[1], X[3]}, xzw[3] = {X[0], X[2], X[3]};
  const float yxy[2] = {Y[0], Y[1]}, yxyw[3] = {Y[0], Y[1], Y[3]};
  float       a[3], b[3];
  mulMv(M1, xy, a);
  mulMv(M2, xyw, b);
  float bias = dotN<2>(a, yxy) * (1.0f / dotN<3>(b, yxyw));
  mulMv(M3, xy, a);
  mulMv(M4, xzw, b);
  const float scale = dotN<2>(a, yxy) * (1.0f / dotN<3>(b, yxyw));
  bias *= fminf(fmaxf(specularColor.y * 50.0f, 0.0f), 1.0f);
  const float sc = fmaxf(0.0f, scale), bi = fmaxf(0.0f, bias);
  return f3(specularColor.x * sc + bi, specularColor.y * sc + bi, specularColor.z * sc + bi);
}

// calculateMotionVector(currWorldPos, prevWorldPos, prevMVP, currentMVP, resolution): mul(float4, float4x4) on the glm bytes
static float2 calculateMotionVector(float4 currWorld, float4 prevWorld, const mat4& prevMVP, const mat4& currMVP, float2 resolution)
{
  const float4 currClip = mul_vM(currWorld, currMVP);
  const float4 prevClip = mul_vM(prevWorld, prevMVP);
  const float2 currNDC = f2(currClip.x / currClip.w, currClip.y / currClip.w);
  const float2 prevNDC = f2(prevClip.x / prevClip.w, prevClip.y / prevClip.w);
  return f2((prevNDC.x - currNDC.x) * 0.5f * resolution.x, (prevNDC.y - currNDC.y) * 0.5f * resolution.y);
}

struct PathTracerState
{
  float3       radiance = f3(0.0f), throughput = f3(1.0f), firstHitPos = f3(1e34f);
  float3       guideAlbedo = f3(0.0f), guideNormal = f3(0.0f);  // GuideScratch (pathtrace_functions.h.slang:79-88): float16_t fields, default 0
  // USE_DLSS_SHADER: the rest of GuideScratch and the first hit's previous-frame position, written on DLSS frames only
  float        guideRoughness = 0.0f;
  float3       firstHitPosPrev = f3(1e34f);
  float3       specAlbedo = f3(0.0f);  // GuideScratch::specularAlbedo (float16_t)
  float        specHitDist = 0.0f;     // GuideScratch::specularHitDist (float16_t)
  bool         captureSpecularHit = false;
  float        lastSamplePdf = DIRAC;
  float2       maxRoughness = f2(0.0f, 0.0f);
  bool         solid = true;
  float        coneWidth = 0.0f, coneSpread = 0.0f;
  int          surfaceDepth = 0;
  bool         isInside = false;
  VolumeMedium medium = {f3(0.0f), f3(0.0f), 0.0f};
  int          scatterBounces = 0;
};
struct BounceScratch
{
  bool   nextEventValid;
  float3 contribution, shadowRayPos, shadowRayDir;
  float  shadowRayDist;
};
enum PathStepResult
{
  eOutOfVolume,
  eVolumeContinue,
  eEarlyContinue,
  eBreak
};

static bool handleVolumeScatter(const VolumeMedium& m, float hitDistance, Ray& ray, float3& throughput, float& lastSamplePdf, uint32_t& seed)
{
  const float3 ext = m.extinction;
  const float3 sc = m.scatterCoefficient;
  const float  maxScatter = maxc(sc);
  if(maxScatter > 0.001f)
  {
    const float maxExt = maxc(ext);
    const float scatterDist = -logf(fmaxf(rnd(seed), 1.0e-10f)) / maxExt;
    if(scatterDist < hitDistance)
    {
      throughput *= f3(1.0f) - (ext - sc) / maxExt;
      ray.o = ray.o + ray.d * scatterDist;
      const float3 wi = ray.d;
      const float  a = rnd(seed), b = rnd(seed);
      ray.d = sampleHenyeyGreenstein(f2(a, b), m.scatterAnisotropy, wi);
      lastSamplePdf = henyeyGreensteinPdf(dot(wi, ray.d), m.scatterAnisotropy);
      return true;
    }
    throughput *= expv((f3(maxExt) - ext) * hitDistance);
    return false;
  }
  throughput *= expv(ext * -hitDistance);
  return false;
}

static float3 volumeScatterNEE(const Ctx& c, const VolumeMedium& m, float3 scatterPos, float3 wi, float3 throughput, uint32_t& seed)
{
  DirectLight dl;
  sampleLights(c, scatterPos, wi, seed, dl, true);
  if(dl.pdf <= 0.0f)  // also rejects DIRAC (-1), exactly like the reference (pathtrace_functions.h.slang:656)
    return f3(0.0f);
  const float cosTheta = dot(wi, dl.direction);
  const float phasePdf = henyeyGreensteinPdf(cosTheta, m.scatterAnisotropy);
  const float misWeight = dl.pdf / (dl.pdf + phasePdf);
  Ray         sr;
  sr.o = scatterPos;
  sr.d = dl.direction;
  sr.tmin = 0.0f;
  sr.tmax = dl.distance;
  float3 shadow = TraceShadow(*c.o, sr, seed, true);
  return throughput * dl.radianceOverPdf * misWeight * phasePdf * shadow;
}

static PathStepResult processVolumeSegment(const Ctx& c, float hitDistance, Ray& ray, PathTracerState& pt, uint32_t& seed)
{
  if(pt.isInside && hasVolumeMedium(pt.medium))
  {
    const float3 wiBefore = ray.d, originBefore = ray.o;
    if(handleVolumeScatter(pt.medium, hitDistance, ray, pt.throughput, pt.lastSamplePdf, seed))
    {
      pt.scatterBounces++;
      pt.coneWidth += pt.coneSpread * length(ray.o - originBefore);
      const float3 nee = volumeScatterNEE(c, pt.medium, ray.o, wiBefore, pt.throughput, seed);
      pt.radiance += nee;
      if(dbgPixel)
        fprintf(stderr, "DBG scatter n=%d o=%.9g %.9g %.9g d=%.9g %.9g %.9g thr=%.9g %.9g %.9g pdf=%.9g nee=%.9g %.9g %.9g seed=%u\n", pt.scatterBounces, ray.o.x, ray.o.y, ray.o.z, ray.d.x,
                ray.d.y, ray.d.z, pt.throughput.x, pt.throughput.y, pt.throughput.z, pt.lastSamplePdf, nee.x, nee.y, nee.z, seed);
      if(pt.scatterBounces >= 64)
      {
        float rrPcont = fminf(maxc(pt.throughput) + 0.001f, 0.95f);
        if(rnd(seed) >= rrPcont)
          return eBreak;
        pt.throughput /= rrPcont;
      }
      return eVolumeContinue;
    }
  }
  return eOutOfVolume;
}

// The DLSS guides of the first hit (gltf_pathtrace.slang:235-255): roughness, previous-frame position and specular albedo.  node is
// the hit's render node, null for the infinite plane.  Kept out of line so that the bounce stays small enough for GCC to inline
// evaluateMaterial into it, as it does without the DLSS captures: plain frames then run the code they ran before the variant.
__attribute__((noinline)) static void dlssFirstHitGuides(const Ctx& c, const PbrMaterial& pbrMat, float3 pos, const b200pt_render_node* node, int rnodeID,
                                                         float3 rayDir, PathTracerState& pt)
{
  pt.guideRoughness = half16(pbrMat.roughness.x);
  // instance motion (:235-241): the surface point in object space, then through the previous frame's objectToWorld
  pt.firstHitPosPrev = pos;
  if(node && c.prevObjectToWorld)
  {
    const float4 objPos = mul_vM(f4(pos.x, pos.y, pos.z, 1.0f), *(const mat4*)node->worldToObject);
    pt.firstHitPosPrev = xyz(mul_vM(f4(objPos.x, objPos.y, objPos.z, 1.0f), *(const mat4*)(c.prevObjectToWorld + 16 * (size_t)rnodeID)));
  }
  // specular albedo (:246-255); pow(x, 2.0) is the correctly rounded square
  const float  q = (pbrMat.ior2 - pbrMat.ior1) / (pbrMat.ior2 + pbrMat.ior1);
  const float  f0FromIor = q * q;
  const float3 clamped = f3(fminf(f0FromIor * pbrMat.specularColor.x, 1.0f), fminf(f0FromIor * pbrMat.specularColor.y, 1.0f),
                            fminf(f0FromIor * pbrMat.specularColor.z, 1.0f));
  const float3 sa = envBRDFApprox2(clamped, pbrMat.roughness.x, dot(pbrMat.N, rayDir));
  pt.specAlbedo = f3(half16(sa.x), half16(sa.y), half16(sa.z));
}

// pathTraceOneBounce (gltf_pathtrace.slang:87-430) with the infinite plane, the shadow catcher and, on DLSS frames, the
// USE_DLSS_SHADER captures (the reference's shader specialization: a plain frame arms no capture and computes no DLSS guide).
// The backplate blur is refused by the frame entry; the visualization modes are not restated.
static PathStepResult pathTraceOneBounce(const Ctx& c, Ray& ray, uint32_t& seed, PathTracerState& pt, BounceScratch& bounce)
{
  Oracle& o = *c.o;
  bounce.nextEventValid = false;
  bounce.contribution = f3(0.0f);
  bounce.shadowRayPos = f3(0.0f);
  bounce.shadowRayDir = f3(0.0f);
  bounce.shadowRayDist = 0.0f;

  HitPayload payload;
  Trace(o, ray, payload, seed);

  const bool firstRay = (pt.surfaceDepth == 0);
  const bool meshHit = payload.hitT != INFINITE_F;
  // checkInfinitePlaneIntersection (pathtrace_functions.h.slang:556-585): the plane y = infinitePlaneDistance, hit from above only,
  // when it is nearer than the geometry hit
  bool     hitInfinitePlane = false;
  HitState planeHit{};
  if(c.fi->flags & B200PT_SCENE_USE_INFINITE_PLANE)
  {
    const float3 normal = f3(0, 1, 0);
    const float  planeHeight = c.fi->infinitePlaneDistance;
    if(!(ray.o.y <= planeHeight))
    {
      const float Dn = dot(ray.d, normal);
      if(!(fabsf(Dn) <= 1e-6f))
      {
        const float On = dot(ray.o, normal);
        const float intersectionDist = (-On + planeHeight) / Dn;
        if(!(intersectionDist <= 0.0f || intersectionDist >= payload.hitT))
        {
          payload.hitT = intersectionDist;
          planeHit.pos = ray.o + ray.d * payload.hitT;
          planeHit.shadowPos = planeHit.pos;
          planeHit.nrm = normal;
          planeHit.geonrm = normal;
          planeHit.tangent = f3(1, 0, 0);
          planeHit.bitangent = f3(0, 0, 1);
          hitInfinitePlane = true;
        }
      }
    }
  }
  if(payload.hitT == INFINITE_F)
  {
    if(firstRay)
    {
      // tryPrimaryMissBackplate (pathtrace_functions.h.slang:944-971)
      pt.solid = false;
      pt.firstHitPos = ray.d;
      pt.firstHitPosPrev = ray.d;
      if(c.fi->flags & B200PT_SCENE_USE_SOLID_BACKGROUND)
      {
        pt.radiance = f3(c.fi->backgroundColor[0], c.fi->backgroundColor[1], c.fi->backgroundColor[2]);
        return eBreak;
      }
    }
    // DLSS: a glossy reflection of the first hit leaves to the sky (gltf_pathtrace.slang:135-143)
    if(pt.captureSpecularHit)
    {
      pt.specHitDist = 65504.0f;
      pt.captureSpecularHit = false;
    }
    float3 envColor;
    float  envPdf;
    sampleEnvironment(c, ray.d, envColor, envPdf);
    float misWeight = computeEnvHitMisWeight(c, pt.lastSamplePdf, envPdf);
    pt.radiance += pt.throughput * misWeight * envColor;
    return eBreak;
  }

  if(dbgPixel)
    fprintf(stderr, "DBG hit t=%.9g rnode=%d prim=%d bary=%.9g %.9g org=%.9g %.9g %.9g dir=%.9g %.9g %.9g seed=%u depth=%d\n", payload.hitT, payload.rnodeID,
            payload.primitiveID, payload.bx, payload.by, ray.o.x, ray.o.y, ray.o.z, ray.d.x, ray.d.y, ray.d.z, seed, pt.surfaceDepth);
  HitState hit = planeHit;
  if(!hitInfinitePlane)
  {
    const b200pt_render_node& rn = o.nodes[payload.rnodeID];
    const Prim&               P = o.prims[payload.rprimID];
    const float3              barys = f3(1.0f - payload.bx - payload.by, payload.bx, payload.by);
    hit = getHitState(P, barys, *(const mat4*)rn.worldToObject, *(const mat4*)rn.objectToWorld, (uint32_t)payload.primitiveID, ray.d);
  }
  (void)meshHit;
  tls.shadedHits++;

  // rayConeWorldFootprint
  float worldFoot;
  {
    float w = pt.coneWidth + pt.coneSpread * payload.hitT;
    worldFoot = w / fmaxf(fabsf(dot(hit.geonrm, -ray.d)), 1e-3f);
  }

  int         materialIndex = -1;
  PbrMaterial pbrMat;
  if(hitInfinitePlane)
  {
    // gltf_pathtrace.slang:169-173: the plane's material replaces the hit's (defaultPbrMaterial(baseColor, metallic, roughness, N, Ng):
    // nvshaders, external -- restated: GGX alpha = roughness^2 like evaluateMaterial, tangent frame from the normal)
    pbrMat = defaultPbrMaterial();
    pbrMat.baseColor = f3(c.fi->infinitePlaneBaseColor[0], c.fi->infinitePlaneBaseColor[1], c.fi->infinitePlaneBaseColor[2]);
    pbrMat.metallic = c.fi->infinitePlaneMetallic;
    const float r = c.fi->infinitePlaneRoughness;
    pbrMat.roughness = f2(r * r, r * r);
    pbrMat.N = hit.nrm;
    pbrMat.Ng = hit.nrm;
    pbrMat.Nc = hit.nrm;
    pbrMat.T = xyz(makeFastTangent(hit.nrm));
    pbrMat.B = cross(pbrMat.N, pbrMat.T);
    // Shadow catcher: the plane shows only the shadows cast on it, over the environment (gltf_pathtrace.slang:175-186 +
    // handleShadowCatcher, pathtrace_functions.h.slang:499-554, followed statement by statement)
    if(c.fi->flags & B200PT_SCENE_INFINITE_PLANE_SHADOW_CATCHER)
    {
      pt.coneWidth = worldFoot;
      DirectLight directLight;
      sampleLights(c, hit.pos, pbrMat.N, seed, directLight, false);
      float3 shadowFactor = f3(1.0f, 1.0f, 1.0f);
      if(dot(directLight.direction, hit.nrm) > 0.0f && directLight.pdf != 0.0f)
      {
        Ray sr;
        sr.o = hit.pos;
        sr.d = directLight.direction;
        sr.tmin = 0.0f;
        sr.tmax = INFINITE_F;
        shadowFactor = TraceShadow(*c.o, sr, seed, false);
      }
      float3 envColor;
      float  envPdf;
      sampleEnvironment(c, ray.d, envColor, envPdf);
      if(shadowFactor.x == 1.0f && shadowFactor.y == 1.0f && shadowFactor.z == 1.0f)
      {
        const float misWeight = computeEnvHitMisWeight(c, pt.lastSamplePdf, envPdf);
        pt.radiance += pt.throughput * misWeight * envColor;
        return eBreak;
      }
      pt.radiance += envColor * shadowFactor;
      pt.radiance -= envColor * (f3(1.0f) - shadowFactor) * c.fi->shadowCatcherDarkenAmount;
      BsdfSampleData sd;
      sd.k1 = -ray.d;
      {
        const float a = rnd(seed), b = rnd(seed), cc = rnd(seed);
        sd.xi = f3(a, b, cc);
      }
      bsdfSampleSimple(sd, pbrMat);
      if(sd.event_type == BSDF_EVENT_ABSORB)
        return eBreak;
      const float3 offsetDir = dot(sd.k2, hit.geonrm) > 0 ? hit.geonrm : -hit.geonrm;
      ray.o = safeOffsetRay(hit.pos, offsetDir);
      ray.d = sd.k2;
      pt.throughput *= sd.bsdf_over_pdf;
      pt.lastSamplePdf = sd.pdf;
      return eEarlyContinue;
    }
  }
  else
  {
    materialIndex = std::max(0, o.nodes[payload.rnodeID].materialID);
    float     texGrad = worldFoot * hit.texelDensity * c.pc->texGradScale;
    MeshState mesh;
    mesh.N = hit.nrm;
    mesh.T = hit.tangent;
    mesh.B = hit.bitangent;
    mesh.Ng = hit.geonrm;
    mesh.tc[0] = hit.uv[0];
    mesh.tc[1] = hit.uv[1];
    mesh.isInside = pt.isInside;
    mesh.texGrad = texGrad;
    mesh.baseColorVertexMul = hit.color;
    pbrMat = evaluateMaterial(o, o.mats[materialIndex], mesh);
  }

  // DLSS: the first surface behind a glossy reflection of the first hit (:216-223); the shadow catcher returned above
  if(pt.captureSpecularHit)
  {
    pt.specHitDist = half16(payload.hitT);
    pt.captureSpecularHit = false;
  }

  if(firstRay)
  {
    pt.firstHitPos = hit.pos;
    // USE_GUIDE_SHADER (gltf_pathtrace.slang:240-263): base colour, shading normal and, on DLSS frames, roughness of the first hit,
    // stored as float16_t by the reference
    pt.guideAlbedo = f3(half16(pbrMat.baseColor.x), half16(pbrMat.baseColor.y), half16(pbrMat.baseColor.z));
    pt.guideNormal = f3(half16(pbrMat.N.x), half16(pbrMat.N.y), half16(pbrMat.N.z));
    if(c.dlss)
      dlssFirstHitGuides(c, pbrMat, hit.pos, hitInfinitePlane ? nullptr : &o.nodes[payload.rnodeID], payload.rnodeID, ray.d, pt);
  }

  pt.maxRoughness = f2(fmaxf(pbrMat.roughness.x, pt.maxRoughness.x), fmaxf(pbrMat.roughness.y, pt.maxRoughness.y));
  pbrMat.roughness = pt.maxRoughness;

  pt.radiance += pbrMat.emissive * pt.throughput;

  if(materialIndex >= 0 && o.mats[materialIndex].unlit > 0)
  {
    pt.radiance += pbrMat.baseColor;
    return eBreak;
  }

  PathStepResult volumeStep = processVolumeSegment(c, payload.hitT, ray, pt, seed);
  if(volumeStep != eOutOfVolume)
    return volumeStep;

  pt.coneWidth = worldFoot;

  DirectLight directLight;
  sampleLights(c, hit.pos, pbrMat.N, seed, directLight, false);

  bounce.nextEventValid = (dot(directLight.direction, hit.nrm) > 0.0f || pbrMat.diffuseTransmissionFactor > 0.0f) && directLight.pdf != 0.0f;
  if(dbgPixel)
    fprintf(stderr, "DBG shade pos=%.9g %.9g %.9g nrm=%.9g %.9g %.9g gn=%.9g %.9g %.9g N=%.9g %.9g %.9g rough=%.9g %.9g metal=%.9g base=%.9g %.9g %.9g L=%.9g %.9g %.9g lpdf=%.9g valid=%d seed=%u\n",
            hit.pos.x, hit.pos.y, hit.pos.z, hit.nrm.x, hit.nrm.y, hit.nrm.z, hit.geonrm.x, hit.geonrm.y, hit.geonrm.z, pbrMat.N.x, pbrMat.N.y, pbrMat.N.z, pbrMat.roughness.x,
            pbrMat.roughness.y, pbrMat.metallic, pbrMat.baseColor.x, pbrMat.baseColor.y, pbrMat.baseColor.z, directLight.direction.x, directLight.direction.y,
            directLight.direction.z, directLight.pdf, (int)bounce.nextEventValid, seed);

  if(bounce.nextEventValid)
  {
    BsdfEvaluateData ev;
    ev.k1 = -ray.d;
    ev.k2 = directLight.direction;
    float a = rnd(seed), b = rnd(seed), cc = rnd(seed);
    ev.xi = f3(a, b, cc);
    bsdfEvaluate(ev, pbrMat);
    if(ev.pdf > 0.0f)
    {
      const float  misWeight = (directLight.pdf == DIRAC) ? 1.0f : directLight.pdf / (directLight.pdf + ev.pdf);
      const float3 w = pt.throughput * directLight.radianceOverPdf * misWeight;
      bounce.contribution += w * ev.bsdf_diffuse;
      bounce.contribution += w * ev.bsdf_glossy;
    }
  }

  {
    BsdfSampleData sd;
    sd.k1 = -ray.d;
    float a = rnd(seed), b = rnd(seed), cc = rnd(seed);
    sd.xi = f3(a, b, cc);
    bsdfSample(sd, pbrMat);
    if(dbgPixel)
      fprintf(stderr, "DBG sample xi=%.9g %.9g %.9g k2=%.9g %.9g %.9g bop=%.9g %.9g %.9g pdf=%.9g ev=%d contrib=%.9g %.9g %.9g\n", sd.xi.x, sd.xi.y, sd.xi.z, sd.k2.x, sd.k2.y,
              sd.k2.z, sd.bsdf_over_pdf.x, sd.bsdf_over_pdf.y, sd.bsdf_over_pdf.z, sd.pdf, sd.event_type, bounce.contribution.x, bounce.contribution.y, bounce.contribution.z);
    pt.throughput *= sd.bsdf_over_pdf;
    ray.d = sd.k2;
    pt.lastSamplePdf = sd.pdf;
    // DLSS: arm the specular hit-distance capture (:370-377)
    if(c.dlss && firstRay && (sd.event_type == BSDF_EVENT_GLOSSY_REFLECTION || sd.event_type == BSDF_EVENT_IMPULSE_REFLECTION))
      pt.captureSpecularHit = true;
    if(sd.event_type != BSDF_EVENT_ABSORB)
    {
      bool   isTransmission = (sd.event_type & BSDF_EVENT_TRANSMISSION) != 0;
      float3 offsetDir = dot(ray.d, hit.geonrm) > 0 ? hit.geonrm : -hit.geonrm;
      ray.o = safeOffsetRay(hit.pos, offsetDir);
      if(isTransmission)
      {
        pt.isInside = !pt.isInside;
        if(pt.isInside)
          pt.medium = makeVolumeMedium(pbrMat);
      }
    }
    else
      pt.surfaceDepth = c.pc->maxDepth;
  }

  const bool   shadowSideForward = dot(directLight.direction, hit.nrm) > 0.0f;
  const float3 shadowOffsetDir = shadowSideForward ? hit.geonrm : -hit.geonrm;
  const float3 shadowOffsetBase = shadowSideForward ? hit.shadowPos : hit.pos;
  bounce.shadowRayPos = safeOffsetRay(shadowOffsetBase, shadowOffsetDir);
  bounce.shadowRayDir = directLight.direction;
  bounce.shadowRayDist = directLight.distance;
  return eOutOfVolume;
}

struct SampleResult
{
  float4 radiance;
  float3 hitPosition;
  float3 guideAlbedo, guideNormal;  // SampleResult::guideOutput (pathtrace_functions.h.slang:94-102)
  float  guideRoughness;            // DLSS frames: the rest of guideOutput and the first hit's previous-frame position
  float3 hitPositionPrev, specAlbedo;
  float  specHitDist;
};

static SampleResult pathTrace(const Ctx& c, Ray ray, uint32_t& seed)
{
  PathTracerState pt;
  pt.coneSpread = c.pc->pixelAngle;
  while(pt.surfaceDepth < c.pc->maxDepth)
  {
    ray.d = normalize(ray.d);
    BounceScratch  bounce;
    PathStepResult step = pathTraceOneBounce(c, ray, seed, pt, bounce);
    if(step == eBreak)
      break;
    if(step == eVolumeContinue || step == eEarlyContinue)
      continue;
    if(bounce.nextEventValid)
    {
      Ray sr;
      sr.o = bounce.shadowRayPos;
      sr.d = bounce.shadowRayDir;
      sr.tmin = 0.0f;
      sr.tmax = bounce.shadowRayDist;
      float3 shadowFactor = TraceShadow(*c.o, sr, seed, false);
      if(dbgPixel)
        fprintf(stderr, "DBG shadow o=%.9g %.9g %.9g d=%.9g %.9g %.9g tmax=%.9g T=%.9g %.9g %.9g\n", sr.o.x, sr.o.y, sr.o.z, sr.d.x, sr.d.y, sr.d.z, sr.tmax, shadowFactor.x,
                shadowFactor.y, shadowFactor.z);
      pt.radiance += bounce.contribution * shadowFactor;
    }
    if(pt.surfaceDepth >= 3)
    {
      float rrPcont = fminf(maxc(pt.throughput) + 0.001f, 0.95f);
      if(rnd(seed) >= rrPcont)
        break;
      pt.throughput /= rrPcont;
    }
    pt.surfaceDepth++;
  }
  SampleResult r;
  r.radiance = f4(pt.radiance, pt.solid ? 1.0f : 0.0f);
  r.hitPosition = pt.firstHitPos;
  r.guideAlbedo = pt.guideAlbedo;
  r.guideNormal = pt.guideNormal;
  r.guideRoughness = pt.guideRoughness;
  r.hitPositionPrev = pt.firstHitPosPrev;
  r.specAlbedo = pt.specAlbedo;
  r.specHitDist = pt.specHitDist;
  return r;
}

static Ray getRay(float2 samplePos, float2 offset, float2 imageSize, const mat4& projI, const mat4& viewI, bool ortho)
{
  const float2 clip = f2((samplePos.x + offset.x) / imageSize.x * 2.0f - 1.0f, (samplePos.y + offset.y) / imageSize.y * 2.0f - 1.0f);
  float4       vc = mul_vM(f4(clip.x, clip.y, -1.0f, 1.0f), projI);
  vc = vc / vc.w;
  Ray ray;
  if(ortho)
  {
    ray.o = xyz(mul_vM(vc, viewI));
    ray.d = normalize(xyz(mul_vM(f4(0, 0, -1, 0), viewI)));
  }
  else
  {
    ray.o = f3(viewI.m[12], viewI.m[13], viewI.m[14]);
    ray.d = normalize(xyz(mul_vM(vc, viewI)) - ray.o);
  }
  ray.tmin = 0.0f;
  ray.tmax = INFINITE_F;
  return ray;
}

static SampleResult samplePixel(const Ctx& c, uint32_t& seed, float2 samplePos, float2 jitter, float2 imageSize)
{
  const mat4& projI = *(const mat4*)c.fi->projInv;
  const mat4& viewI = *(const mat4*)c.fi->viewInv;
  const bool  ortho = (c.fi->flags & B200PT_SCENE_IS_ORTHOGRAPHIC) != 0;
  Ray         ray = getRay(samplePos, jitter, imageSize, projI, viewI, ortho);
  if(!ortho)
  {
    float3 focalPoint = ray.d * c.pc->focalDistance;
    float  cam_r1 = rnd(seed) * M_TWO_PI_F;
    float  cam_r2 = rnd(seed) * c.pc->aperture;
    float4 cam_right = mul_Mv(viewI, f4(1, 0, 0, 0));
    float4 cam_up = mul_Mv(viewI, f4(0, 1, 0, 0));
    float3 rap = (xyz(cam_right) * cosf(cam_r1) + xyz(cam_up) * sinf(cam_r1)) * sqrtf(cam_r2);
    float3 finalDir = normalize(focalPoint - rap);
    ray.o += rap;
    ray.d = finalDir;
  }
  SampleResult sr = pathTrace(c, ray, seed);
  float        lum = (sr.radiance.x + sr.radiance.y + sr.radiance.z) * (1.0f / 3.0f);
  if(lum > c.pc->fireflyClampThreshold)
    sr.radiance = sr.radiance * (c.pc->fireflyClampThreshold / lum);
  return sr;
}

static float2 sampleGaussian(float2 u)
{
  const float r = sqrtf(-2.0f * logf(fmaxf(1e-38f, u.x)));
  const float theta = 2.0f * M_PI_F * u.y;
  return f2(r * cosf(theta), r * sinf(theta));
}

// TraceLow (raytracer_interface.h.slang:124-137): every triangle opaque, no culling -> nearest hit of both trees
static int traceLowObjectId(Oracle& o, const Ray& ray)
{
  Hit  ho, ha;
  const bool a = nextHit(o, o.treeOpaque, ray, false, 0.f, 0u, false, ho);
  const bool b = !o.treeAlpha.bvh.empty() && nextHit(o, o.treeAlpha, ray, false, 0.f, 0u, false, ha);
  if(!a && !b)
    return 0;
  const Hit& h = (a && (!b || ho.t < ha.t || (ho.t == ha.t && ho.tri < ha.tri))) ? ho : ha;
  return (int)o.tris[h.tri].rnode + 1;
}

// nvshaders' compressUnitVec (external): octahedral 2 x 16-bit encoding (Engelhardt & Dachsbacher 2008), restated
static uint32_t compressUnitVec(float3 nv)
{
  if(!(fabsf(nv.x) < 3.0e38f))
    return ~0u;
  const float d = 32767.0f / (fabsf(nv.x) + fabsf(nv.y) + fabsf(nv.z));
  int         x = (int)roundf(nv.x * d), y = (int)roundf(nv.y * d);
  if(nv.z < 0.0f)
  {
    const int maskx = x >> 31, masky = y >> 31;
    const int tmp = 32767 + maskx + masky, tmpx = x;
    x = (tmp - (y ^ masky)) ^ maskx;
    y = (tmp - (tmpx ^ maskx)) ^ masky;
  }
  const uint32_t packed = ((uint32_t)(y + 32767) << 16) | (uint32_t)(x + 32767);
  return packed == ~0u ? ~1u : packed;
}

// the DLSS guide planes of one pixel
struct DlssOut
{
  uint32_t* albedo;       // RGBA8 UNORM
  uint16_t* specAlbedo;   // RGBA16F
  uint16_t* normalRough;  // RGBA16F
  uint16_t* motion;       // RG16F
  uint16_t* depth;        // R16F
  uint16_t* specHitDist;  // R16F
};

// processPixel (gltf_pathtrace.slang:546-651).  A DLSS frame (dlss non-null, numSamples == 1) samples at the frame's jitter, replaces
// the image and writes the guide planes.
static void processPixel(const Ctx& c, int x, int y, float* px, uint32_t* objectId, float* ndcDepth, float* guide, const DlssOut* dlss)
{
  const float2 imageSize = f2(c.fi->imageSize[0], c.fi->imageSize[1]);
  const float2 samplePos = f2((float)x, (float)y);
  uint32_t     seed = xxhash32((uint32_t)x, (uint32_t)y, (uint32_t)c.pc->frameCount);
  dbgPixel = ((float)x == c.pc->mouseCoord[0] && (float)y == c.pc->mouseCoord[1]);
  const bool   firstFrame = (c.pc->flags & B200PT_PT_FIRST_FRAME) != 0;
  float2       jitter = f2(0.5f, 0.5f);
  if(c.dlss)
    jitter = f2(0.5f + c.fi->jitter[0], 0.5f + c.fi->jitter[1]);  // the frame's DLSS jitter; no Gaussian draw (gltf_pathtrace.slang:568-572)
  else
  {
    float  a = rnd(seed), b = rnd(seed);
    float2 g = sampleGaussian(f2(a, b));
    jitter = jitter + g * 0.4246609f;
  }
  tls.paths++;
  SampleResult sr = samplePixel(c, seed, samplePos, jitter, imageSize);
  float4       pixelColor = sr.radiance;
  for(int s = 1; s < c.pc->numSamples; s++)
  {
    float a = rnd(seed), b = rnd(seed);
    jitter = f2(a, b);
    tls.paths++;
    sr = samplePixel(c, seed, samplePos, jitter, imageSize);
    pixelColor += sr.radiance;
  }
  pixelColor = pixelColor / (float)c.pc->numSamples;
  if(firstFrame && (objectId || ndcDepth))
  {
    // gltf_pathtrace.slang:600-616: NDC depth of the LAST sample's first hit, object id of the selection ray
    const bool hasSolidHit = sr.radiance.w > 0.0f;
    float      d = 1.0f;
    if(hasSolidHit)
    {
      const float4 clip = mul_vM(f4(sr.hitPosition.x, sr.hitPosition.y, sr.hitPosition.z, 1.0f), *(const mat4*)c.fi->viewProjMatrix);
      d = clip.z / clip.w;
    }
    if(ndcDepth)
      *ndcDepth = d;
    if(objectId)
    {
      const bool ortho = (c.fi->flags & B200PT_SCENE_IS_ORTHOGRAPHIC) != 0;
      const Ray  ray = getRay(samplePos, f2(0.5f, 0.5f), imageSize, *(const mat4*)c.fi->projInv, *(const mat4*)c.fi->viewInv, ortho);
      *objectId = (uint32_t)traceLowObjectId(*c.o, ray);
    }
  }
  if(guide && (c.pc->flags & B200PT_PT_USE_OPTIX_DENOISER))
  {
    // gltf_pathtrace.slang:653-670: eOptixAlbedoNormal = (guide albedo of the LAST sample, compressed camera-space normal);
    // mul(float3x3(viewMatrix), n) on the glm bytes is M_glm^T * n (SURVEY.md section 8, convention note)
    float3 camN = f3(0.0f, 0.0f, 1.0f);
    if(sr.radiance.w > 0.0f)
    {
      const float* m = c.fi->viewMatrix;
      const float3 n = sr.guideNormal;
      camN = normalize(f3((m[0] * n.x + m[1] * n.y) + m[2] * n.z, (m[4] * n.x + m[5] * n.y) + m[6] * n.z, (m[8] * n.x + m[9] * n.y) + m[10] * n.z));
    }
    const uint32_t packed = compressUnitVec(camN);
    guide[0] = sr.guideAlbedo.x;
    guide[1] = sr.guideAlbedo.y;
    guide[2] = sr.guideAlbedo.z;
    memcpy(&guide[3], &packed, 4);
  }
  if(dlss)
  {
    // gltf_pathtrace.slang:628-651
    const bool   hasSolidHit = sr.radiance.w > 0.0f;
    float        d = 1.0f;
    const mat4&  vp = *(const mat4*)c.fi->viewProjMatrix;
    if(hasSolidHit)
    {
      const float4 clip = mul_vM(f4(sr.hitPosition.x, sr.hitPosition.y, sr.hitPosition.z, 1.0f), vp);
      d = clip.z / clip.w;
    }
    const float  hitW = hasSolidHit ? 1.0f : 0.0f;
    const float2 mv = calculateMotionVector(f4(sr.hitPosition.x, sr.hitPosition.y, sr.hitPosition.z, hitW),
                                            f4(sr.hitPositionPrev.x, sr.hitPositionPrev.y, sr.hitPositionPrev.z, hitW), *(const mat4*)c.fi->prevMVP, vp, imageSize);
    *dlss->depth = halfBits(d);
    dlss->motion[0] = halfBits(mv.x);
    dlss->motion[1] = halfBits(mv.y);
    const float nr[4] = {sr.guideNormal.x, sr.guideNormal.y, sr.guideNormal.z, sr.guideRoughness};
    for(int k = 0; k < 4; k++)
      dlss->normalRough[k] = halfBits(nr[k]);
    *dlss->albedo = unorm8(sr.guideAlbedo.x) | (unorm8(sr.guideAlbedo.y) << 8) | (unorm8(sr.guideAlbedo.z) << 16) | (unorm8(hitW) << 24);
    const float sa[4] = {sr.specAlbedo.x, sr.specAlbedo.y, sr.specAlbedo.z, 1.0f};
    for(int k = 0; k < 4; k++)
      dlss->specAlbedo[k] = halfBits(sa[k]);
    *dlss->specHitDist = halfBits(sr.specHitDist);
  }
  if(firstFrame || c.dlss)
  {
    px[0] = pixelColor.x;
    px[1] = pixelColor.y;
    px[2] = pixelColor.z;
    px[3] = pixelColor.w;
  }
  else
  {
    const float total = (float)c.pc->totalSamples, n = (float)c.pc->numSamples;
    const float after = (float)(c.pc->totalSamples + c.pc->numSamples);
    px[0] = (px[0] * total + pixelColor.x * n) / after;
    px[1] = (px[1] * total + pixelColor.y * n) / after;
    px[2] = (px[2] * total + pixelColor.z * n) / after;
    px[3] = (px[3] * total + pixelColor.w * n) / after;
  }
}

}  // namespace

// =================================================================================================
// C API (ctypes; tests only)
// =================================================================================================
extern "C" {

// SceneOmm::create analogue (src/gltf_scene_omm.cpp): same arrays as b200pt_set_opacity_micromaps; call before or after oracle_set_scene
int oracle_set_opacity_micromaps(void* h, const b200pt_micromap* micromaps, uint32_t numMicromaps, const b200pt_primitive_omm* prims, uint32_t numPrims)
{
  Oracle& o = *(Oracle*)h;
  o.micromaps.clear();
  o.primOmm.clear();
  o.ommOfPrim.clear();
  if(numPrims == 0)
    return 0;
  o.micromaps.resize(numMicromaps);
  for(uint32_t m = 0; m < numMicromaps; m++)
  {
    o.micromaps[m].data.assign(micromaps[m].data, micromaps[m].data + micromaps[m].dataSize);
    o.micromaps[m].tris.assign(micromaps[m].triangles, micromaps[m].triangles + micromaps[m].numTriangles);
  }
  for(uint32_t i = 0; i < numPrims; i++)
  {
    if(prims[i].micromap >= numMicromaps)
      return -1;
    Oracle::PrimOmm po;
    po.micromap = prims[i].micromap;
    po.base = prims[i].baseTriangle;
    po.hasIdx = prims[i].indices != nullptr;
    if(prims[i].indices)
      po.idx.assign(prims[i].indices, prims[i].indices + prims[i].numIndices);
    if(o.ommOfPrim.size() <= prims[i].renderPrimID)
      o.ommOfPrim.resize((size_t)prims[i].renderPrimID + 1, -1);
    o.ommOfPrim[prims[i].renderPrimID] = (int)o.primOmm.size();
    o.primOmm.push_back(std::move(po));
  }
  return 0;
}

void* oracle_create() { return new Oracle(); }
void  oracle_destroy(void* h) { delete(Oracle*)h; }

int oracle_set_scene(void* h, const b200pt_scene_desc* s)
{
  Oracle& o = *(Oracle*)h;
  o.nodes.assign(s->renderNodes, s->renderNodes + s->numRenderNodes);
  o.visible.assign(s->numRenderNodes, 1);
  if(s->renderNodeVisible)
    o.visible.assign(s->renderNodeVisible, s->renderNodeVisible + s->numRenderNodes);
  o.prims.clear();
  o.prims.resize(s->numRenderPrimitives);
  for(uint32_t i = 0; i < s->numRenderPrimitives; i++)
  {
    const b200pt_render_primitive& p = s->renderPrimitives[i];
    Prim&                          P = o.prims[i];
    P.ntri = p.triangleCount;
    P.nvert = p.vertexCount;
    P.idx.assign(p.indices, p.indices + (size_t)p.triangleCount * 3);
    P.pos.assign(p.positions, p.positions + (size_t)p.vertexCount * 3);
    if(p.normals)
      P.nrm.assign(p.normals, p.normals + (size_t)p.vertexCount * 3);
    if(p.tangents)
      P.tan.assign(p.tangents, p.tangents + (size_t)p.vertexCount * 4);
    if(p.texCoords[0])
      P.uv0.assign(p.texCoords[0], p.texCoords[0] + (size_t)p.vertexCount * 2);
    if(p.texCoords[1])
      P.uv1.assign(p.texCoords[1], p.texCoords[1] + (size_t)p.vertexCount * 2);
    if(p.colors)
      P.col.assign(p.colors, p.colors + p.vertexCount);
  }
  o.mats.assign(s->materials, s->materials + s->numMaterials);
  if(o.mats.empty())
    return -1;
  o.texInfos.assign(s->textureInfos, s->textureInfos + s->numTextureInfos);
  o.textures.clear();
  o.textures.resize(s->numTextures);
  {
    std::atomic<uint32_t>    nextTex{0};
    std::vector<std::thread> workers;
    auto                     job = [&]() {
      for(uint32_t i = nextTex.fetch_add(1); i < s->numTextures; i = nextTex.fetch_add(1))
        buildTexture(o.textures[i], s->textures[i]);
    };
    const unsigned nt = std::max(1u, std::min(std::thread::hardware_concurrency(), s->numTextures));
    for(unsigned t = 1; t < nt; t++)
      workers.emplace_back(job);
    job();
    for(auto& t : workers)
      t.join();
  }
  o.lights.assign(s->lights, s->lights + s->numLights);

  // flatten: one world-space triangle per (visible render node, triangle), node order then triangle
  // order — defines the global triangle id used for tie-breaking (same order in the CUDA path)
  o.tris.clear();
  for(uint32_t n = 0; n < s->numRenderNodes; n++)
  {
    if(!o.visible[n])
      continue;
    const b200pt_render_node&    node = o.nodes[n];
    const Prim&                  P = o.prims[node.renderPrimID];
    const b200pt_shade_material& m = o.mats[std::max(0, node.materialID)];
    // getInstanceFlag (src/gltf_scene_rtx.cpp:271-295)
    uint32_t flags = 0;
    if(m.transmissionFactor == 0.0f && m.alphaMode == 0 && m.diffuseTransmissionFactor == 0.0f)
      flags |= TRI_OPAQUE;
    if(m.doubleSided == 1 || m.thicknessFactor > 0.0f || m.transmissionFactor > 0.0f)
      flags |= TRI_NOCULL;
    const mat4&  M = *(const mat4*)node.objectToWorld;
    const float* a = M.m;
    const float  det = a[0] * (a[5] * a[10] - a[9] * a[6]) - a[4] * (a[1] * a[10] - a[9] * a[2]) + a[8] * (a[1] * a[6] - a[5] * a[2]);
    const bool   mirrored = det < 0.0f;
    for(uint32_t t = 0; t < P.ntri; t++)
    {
      float3 p0 = xfPoint(M, ld3(P.pos, P.idx[t * 3])), p1 = xfPoint(M, ld3(P.pos, P.idx[t * 3 + 1])), p2 = xfPoint(M, ld3(P.pos, P.idx[t * 3 + 2]));
      FlatTri T;
      T.rnode = n;
      T.prim = t;
      T.flags = flags;
      if(mirrored)
      {
        std::swap(p1, p2);
        T.flags |= TRI_FLIPPED;
      }
      T.v0 = p0;
      T.e1 = p1 - p0;
      T.e2 = p2 - p0;
      o.tris.push_back(T);
    }
  }
  std::vector<uint32_t> idsO, idsA;
  for(uint32_t i = 0; i < (uint32_t)o.tris.size(); i++)
    ((o.tris[i].flags & TRI_OPAQUE) ? idsO : idsA).push_back(i);
  buildBvh(o, o.treeOpaque, idsO);
  buildBvh(o, o.treeAlpha, idsA);
  return 0;
}

int oracle_set_environment(void* h, const float* rgb, int w, int hh, float* integral)
{
  Oracle& o = *(Oracle*)h;
  setEnvironment(o, rgb, w, hh);
  if(integral)
    *integral = o.envIntegral;
  return 0;
}

// copies out rgba (w*h*4), alias (w*h), q (w*h); any may be NULL
int oracle_get_environment(void* h, float* rgba, uint32_t* alias, float* q)
{
  Oracle& o = *(Oracle*)h;
  size_t  n = (size_t)o.envW * o.envH;
  if(rgba)
    memcpy(rgba, o.envRgba.data(), n * 16);
  if(alias)
    memcpy(alias, o.envAlias.data(), n * 4);
  if(q)
    memcpy(q, o.envQ.data(), n * 4);
  return 0;
}

// Renders rows [y0, y0+rows) of the frame into accum (rows x width x 4 floats, tile-local): the running mean of processPixel, or the
// replaced image of a DLSS frame (pc carries B200PT_PT_USE_DLSS).  The other outputs are tile-local and may be null:
//   objectId / ndcDepth (rows x width): the frame-0 outputs of processPixel;
//   guide (rows x width x 4 floats): OutputImage::eOptixAlbedoNormal, written when pc carries B200PT_PT_USE_OPTIX_DENOISER;
//   prevObjectToWorld: the previous frame's objectToWorld, 16 floats per render node, for a DLSS frame's instance motion; null gives
//   camera-only motion;
//   dlssPlanes: six pointers to the DLSS guide planes (rows x width each): albedo RGBA8, specular albedo RGBA16F, normal / roughness
//   RGBA16F, motion RG16F, depth R16F, specular hit distance R16F.
// Like b200pt_render_frame, B200PT_E_INVALID for a DLSS frame without the planes or with numSamples != 1, and for planes with a plain
// frame.
int oracle_render_frame(void* h, const b200pt_frame_info* fi, const b200pt_push_constant* pc, float* accum, uint32_t* objectId, float* ndcDepth, float* guide,
                        const float* prevObjectToWorld, void* const* dlssPlanes, int y0, int rows, int nthreads)
{
  Oracle& o = *(Oracle*)h;
  if(!(fi->flags & B200PT_SCENE_USE_HDR_ENVIRONMENT) || o.envW == 0)
    return B200PT_E_UNSUPPORTED;
  if(fi->envBlur > 0.0f && !(fi->flags & B200PT_SCENE_USE_SOLID_BACKGROUND))
    return B200PT_E_UNSUPPORTED;  // tryPrimaryMissBackplate's smoothHDRBlur (nvshaders, external)
  const bool dlss = (pc->flags & B200PT_PT_USE_DLSS) != 0;
  if(dlss != (dlssPlanes != nullptr) || (dlss && pc->numSamples != 1))
    return B200PT_E_INVALID;
  const Ctx c{&o, fi, pc, dlss, prevObjectToWorld};
  const int W = (int)fi->imageSize[0];
  nthreads = std::max(1, nthreads);
  std::atomic<int>         next{0};
  std::vector<std::thread> th;
  auto                     work = [&]() {
    for(;;)
    {
      int r = next.fetch_add(1);
      if(r >= rows)
        break;
      for(int x = 0; x < W; x++)
      {
        const size_t  p = (size_t)r * W + x;
        const DlssOut d = dlss ? DlssOut{(uint32_t*)dlssPlanes[0] + p, (uint16_t*)dlssPlanes[1] + 4 * p, (uint16_t*)dlssPlanes[2] + 4 * p,
                                         (uint16_t*)dlssPlanes[3] + 2 * p, (uint16_t*)dlssPlanes[4] + p, (uint16_t*)dlssPlanes[5] + p}
                               : DlssOut{};
        processPixel(c, x, y0 + r, accum + p * 4, objectId ? objectId + p : nullptr, ndcDepth ? ndcDepth + p : nullptr, guide ? guide + p * 4 : nullptr,
                     dlss ? &d : nullptr);
      }
    }
    o.stats.merge();
  };
  for(int t = 1; t < nthreads; t++)
    th.emplace_back(work);
  work();
  for(auto& t : th)
    t.join();
  return 0;
}

int oracle_trace_closest(void* h, const float* rays, uint32_t n, float* hits, uint32_t* seeds)
{
  Oracle& o = *(Oracle*)h;
  for(uint32_t i = 0; i < n; i++)
  {
    Ray r;
    r.o = f3(rays[i * 8], rays[i * 8 + 1], rays[i * 8 + 2]);
    r.tmin = rays[i * 8 + 3];
    r.d = f3(rays[i * 8 + 4], rays[i * 8 + 5], rays[i * 8 + 6]);
    r.tmax = rays[i * 8 + 7];
    uint32_t   seed = seeds ? seeds[i] : 0;
    HitPayload p;
    Trace(o, r, p, seed);
    if(seeds)
      seeds[i] = seed;
    float* out = hits + (size_t)i * 6;
    out[0] = p.hitT;
    memcpy(out + 1, &p.rnodeID, 4);
    memcpy(out + 2, &p.rprimID, 4);
    memcpy(out + 3, &p.primitiveID, 4);
    out[4] = p.bx;
    out[5] = p.by;
  }
  o.stats.merge();
  return 0;
}

int oracle_trace_shadow(void* h, const float* rays, uint32_t n, float* transmission, uint32_t* seeds)
{
  Oracle& o = *(Oracle*)h;
  for(uint32_t i = 0; i < n; i++)
  {
    Ray r;
    r.o = f3(rays[i * 8], rays[i * 8 + 1], rays[i * 8 + 2]);
    r.tmin = rays[i * 8 + 3];
    r.d = f3(rays[i * 8 + 4], rays[i * 8 + 5], rays[i * 8 + 6]);
    r.tmax = rays[i * 8 + 7];
    uint32_t seed = seeds ? seeds[i] : 0;
    float3   t = TraceShadow(o, r, seed, false);
    if(seeds)
      seeds[i] = seed;
    transmission[i * 3] = t.x;
    transmission[i * 3 + 1] = t.y;
    transmission[i * 3 + 2] = t.z;
  }
  o.stats.merge();
  return 0;
}

// multi-threaded closest-hit traversal for the CPU-baseline timing (no alpha seeds)
int oracle_trace_closest_mt(void* h, const float* rays, uint32_t n, float* hits, int nthreads)
{
  nthreads = std::max(1, nthreads);
  std::vector<std::thread> th;
  uint32_t                 chunk = (n + nthreads - 1) / nthreads;
  for(int t = 0; t < nthreads; t++)
  {
    uint32_t a = std::min(n, t * chunk), b = std::min(n, a + chunk);
    th.emplace_back([=]() { oracle_trace_closest(h, rays + (size_t)a * 8, b - a, hits + (size_t)a * 6, nullptr); });
  }
  for(auto& t : th)
    t.join();
  return 0;
}

// BSDF unit hooks. in: 48 floats per item (packing: vk_gltf_renderer_b200/bsdf_io.py)
static PbrMaterial unpackMat(const float* p)
{
  PbrMaterial m = defaultPbrMaterial();
  m.baseColor = f3(p[0], p[1], p[2]);
  m.roughness = f2(p[3], p[4]);
  m.metallic = p[5];
  m.N = f3(p[6], p[7], p[8]);
  m.T = f3(p[9], p[10], p[11]);
  m.B = f3(p[12], p[13], p[14]);
  m.Ng = f3(p[15], p[16], p[17]);
  m.ior1 = p[18];
  m.ior2 = p[19];
  m.specular = p[20];
  m.specularColor = f3(p[21], p[22], p[23]);
  m.transmission = p[24];
  m.thickness = p[25];
  m.clearcoat = p[26];
  m.clearcoatRoughness = p[27];
  m.Nc = m.N;
  m.iridescence = p[28];
  m.iridescenceIor = p[29];
  m.iridescenceThickness = p[30];
  m.sheenColor = f3(p[31], p[32], p[33]);
  m.sheenRoughness = p[34];
  m.diffuseTransmissionFactor = p[35];
  m.diffuseTransmissionColor = f3(p[36], p[37], p[38]);
  return m;
}

// out per item: bsdf_diffuse(3) bsdf_glossy(3) pdf(1) pad(1)
int oracle_bsdf_eval(const float* in, uint32_t n, float* out)
{
  for(uint32_t i = 0; i < n; i++)
  {
    const float*     p = in + (size_t)i * 48;
    PbrMaterial      m = unpackMat(p);
    BsdfEvaluateData d;
    d.k1 = f3(p[39], p[40], p[41]);
    d.k2 = f3(p[42], p[43], p[44]);
    d.xi = f3(p[45], p[46], p[47]);
    bsdfEvaluate(d, m);
    float* q = out + (size_t)i * 8;
    q[0] = d.bsdf_diffuse.x;
    q[1] = d.bsdf_diffuse.y;
    q[2] = d.bsdf_diffuse.z;
    q[3] = d.bsdf_glossy.x;
    q[4] = d.bsdf_glossy.y;
    q[5] = d.bsdf_glossy.z;
    q[6] = d.pdf;
    q[7] = 0.f;
  }
  return 0;
}

// out per item: k2(3) bsdf_over_pdf(3) pdf(1) event(1, as float)
int oracle_bsdf_sample(const float* in, uint32_t n, float* out)
{
  for(uint32_t i = 0; i < n; i++)
  {
    const float*   p = in + (size_t)i * 48;
    PbrMaterial    m = unpackMat(p);
    BsdfSampleData d;
    d.k1 = f3(p[39], p[40], p[41]);
    d.xi = f3(p[45], p[46], p[47]);
    bsdfSample(d, m);
    float* q = out + (size_t)i * 8;
    q[0] = d.k2.x;
    q[1] = d.k2.y;
    q[2] = d.k2.z;
    q[3] = d.bsdf_over_pdf.x;
    q[4] = d.bsdf_over_pdf.y;
    q[5] = d.bsdf_over_pdf.z;
    q[6] = d.pdf;
    q[7] = (float)d.event_type;
  }
  return 0;
}

// the shadow catcher's continuation BSDF evaluated (bsdfEvaluateSimple); same packing and output as oracle_bsdf_eval
int oracle_bsdf_eval_simple(const float* in, uint32_t n, float* out)
{
  for(uint32_t i = 0; i < n; i++)
  {
    const float*     p = in + (size_t)i * 48;
    PbrMaterial      m = unpackMat(p);
    BsdfEvaluateData d;
    d.k1 = f3(p[39], p[40], p[41]);
    d.k2 = f3(p[42], p[43], p[44]);
    d.xi = f3(p[45], p[46], p[47]);
    bsdfEvaluateSimple(d, m);
    float* q = out + (size_t)i * 8;
    q[0] = d.bsdf_diffuse.x;
    q[1] = d.bsdf_diffuse.y;
    q[2] = d.bsdf_diffuse.z;
    q[3] = d.bsdf_glossy.x;
    q[4] = d.bsdf_glossy.y;
    q[5] = d.bsdf_glossy.z;
    q[6] = d.pdf;
    q[7] = 0.f;
  }
  return 0;
}

// the shadow catcher's continuation BSDF (bsdfSampleSimple); same packing and output as oracle_bsdf_sample
int oracle_bsdf_sample_simple(const float* in, uint32_t n, float* out)
{
  for(uint32_t i = 0; i < n; i++)
  {
    const float*   p = in + (size_t)i * 48;
    PbrMaterial    m = unpackMat(p);
    BsdfSampleData d;
    d.k1 = f3(p[39], p[40], p[41]);
    d.xi = f3(p[45], p[46], p[47]);
    bsdfSampleSimple(d, m);
    float* q = out + (size_t)i * 8;
    q[0] = d.k2.x;
    q[1] = d.k2.y;
    q[2] = d.k2.z;
    q[3] = d.bsdf_over_pdf.x;
    q[4] = d.bsdf_over_pdf.y;
    q[5] = d.bsdf_over_pdf.z;
    q[6] = d.pdf;
    q[7] = (float)d.event_type;
  }
  return 0;
}

// DLSS arithmetic on records: EnvBRDFApprox2 on (specular colour xyz, alpha, NoV) -> rgb; calculateMotionVector on (current xyzw,
// previous xyzw, resolution xy) with the two view-projection matrices (glm order) -> pixel motion xy
// Henyey-Greenstein phase function and the multiscatter-to-single-scatter albedo fit, for tests/test_phase_sampling.py
//   oracle_hg_sample: in [n][6] (xi.x, xi.y, g, wi.xyz) -> out [n][3] sampleHenyeyGreenstein
//   oracle_hg_pdf:    in [n][2] (cos theta, g)          -> out [n]    henyeyGreensteinPdf
//   oracle_ssa:       in [n] rho                         -> out [n]    multiToSingleScatterAlbedo
int oracle_hg_sample(const float* in, uint32_t n, float* out)
{
  for(uint32_t i = 0; i < n; i++)
  {
    const float* p = in + 6 * (size_t)i;
    const float3 d = sampleHenyeyGreenstein(f2(p[0], p[1]), p[2], f3(p[3], p[4], p[5]));
    out[3 * i + 0] = d.x;
    out[3 * i + 1] = d.y;
    out[3 * i + 2] = d.z;
  }
  return 0;
}
int oracle_hg_pdf(const float* in, uint32_t n, float* out)
{
  for(uint32_t i = 0; i < n; i++)
    out[i] = henyeyGreensteinPdf(in[2 * i], in[2 * i + 1]);
  return 0;
}
int oracle_ssa(const float* in, uint32_t n, float* out)
{
  for(uint32_t i = 0; i < n; i++)
    out[i] = multiToSingleScatterAlbedo(f3(in[i])).x;
  return 0;
}
int oracle_dlss_env_brdf_approx2(const float* in, uint32_t n, float* out)
{
  for(uint32_t i = 0; i < n; i++)
  {
    const float* p = in + 5 * (size_t)i;
    const float3 r = envBRDFApprox2(f3(p[0], p[1], p[2]), p[3], p[4]);
    out[3 * i + 0] = r.x;
    out[3 * i + 1] = r.y;
    out[3 * i + 2] = r.z;
  }
  return 0;
}
int oracle_dlss_motion_vector(const float* in, uint32_t n, const float* prevMVP, const float* currMVP, float* out)
{
  for(uint32_t i = 0; i < n; i++)
  {
    const float* p = in + 10 * (size_t)i;
    const float2 mv = calculateMotionVector(f4(p[0], p[1], p[2], p[3]), f4(p[4], p[5], p[6], p[7]), *(const mat4*)prevMVP, *(const mat4*)currMVP, f2(p[8], p[9]));
    out[2 * i + 0] = mv.x;
    out[2 * i + 1] = mv.y;
  }
  return 0;
}

int oracle_get_stats(void* h, uint64_t* out6)
{
  Oracle& o = *(Oracle*)h;
  out6[0] = o.stats.closestRays;
  out6[1] = o.stats.shadowRays;
  out6[2] = o.stats.shadedHits;
  out6[3] = o.stats.paths;
  out6[4] = o.stats.nodes;
  out6[5] = o.stats.tris;
  return 0;
}
int oracle_reset_stats(void* h)
{
  Oracle& o = *(Oracle*)h;
  o.stats.closestRays = o.stats.shadowRays = o.stats.shadedHits = o.stats.paths = o.stats.nodes = o.stats.tris = 0;
  return 0;
}
int oracle_num_tris(void* h) { return (int)((Oracle*)h)->tris.size(); }

// small utility hooks for known-answer tests
uint32_t oracle_xxhash32(uint32_t x, uint32_t y, uint32_t z) { return xxhash32(x, y, z); }
float    oracle_rand(uint32_t* seed) { return rnd(*seed); }
void     oracle_safe_offset_ray(const float* p, const float* d, float* out)
{
  float3 r = safeOffsetRay(f3(p[0], p[1], p[2]), f3(d[0], d[1], d[2]));
  out[0] = r.x;
  out[1] = r.y;
  out[2] = r.z;
}
// texture sampling hook: tex index, uv, isotropic gradient g (0 => level 0)
void oracle_sample_texture(void* h, int tex, float u, float v, float g, float* rgba)
{
  Oracle& o = *(Oracle*)h;
  float4  r = sampleTexture(o.textures[tex], f2(u, v), f2(g, 0), f2(0, g), g > 0.0f);
  rgba[0] = r.x;
  rgba[1] = r.y;
  rgba[2] = r.z;
  rgba[3] = r.w;
}
// texture unit-test hook, the records of b200pt_texture_lookup (vk_gltf_renderer_b200/tex_io.py): texture-info slot, mode
// (0 getTexture, 1 sampleLevel0 on the selected texture coordinate), tc0.xy, tc1.xy, texGrad, pad -> rgba
int oracle_texture_lookup(void* h, const float* in, uint32_t n, float* out)
{
  Oracle& o = *(Oracle*)h;
  for(uint32_t i = 0; i < n; i++)
  {
    const float* p = in + (size_t)i * 8;
    if(!(p[0] >= 0.0f && p[0] < (float)o.texInfos.size() && p[0] == floorf(p[0])) || !(p[1] == 0.0f || p[1] == 1.0f))
      return -1;
    const b200pt_texture_info& ti = o.texInfos[(size_t)p[0]];
    const float2               tc[2] = {f2(p[2], p[3]), f2(p[4], p[5])};
    const float4               r = p[1] == 0.0f ? getTexture(o, ti, tc, p[6]) : sampleLevel0(o, ti, tc[ti.texCoord]);
    float*                     q = out + (size_t)i * 4;
    q[0] = r.x;
    q[1] = r.y;
    q[2] = r.z;
    q[3] = r.w;
  }
  return 0;
}

// hit-state unit hook: per record the closest hit, getHitState, the ray-cone texture gradient and evaluateMaterial, called as
// the bounce calls them (layout: vk_gltf_renderer_b200/shade_io.py)
static void putShadeField(float* q, int at, float3 v)
{
  q[at] = v.x;
  q[at + 1] = v.y;
  q[at + 2] = v.z;
}
int oracle_shade_state(void* h, const float* in, uint32_t n, float* out, uint32_t* seeds)
{
  Oracle& o = *(Oracle*)h;
  for(uint32_t i = 0; i < n; i++)
  {
    const float* p = in + (size_t)i * 16;
    float*       q = out + (size_t)i * 96;
    Ray          r;
    r.o = f3(p[0], p[1], p[2]);
    r.tmin = p[3];
    r.d = f3(p[4], p[5], p[6]);
    r.tmax = p[7];
    uint32_t   seed = seeds ? seeds[i] : 0;
    HitPayload pl;
    Trace(o, r, pl, seed);
    if(seeds)
      seeds[i] = seed;
    std::fill(q, q + 96, 0.0f);
    q[0] = pl.hitT;
    q[1] = (float)pl.rnodeID;
    q[2] = (float)pl.rprimID;
    q[3] = (float)pl.primitiveID;
    if(pl.hitT == INFINITE_F)
      continue;
    q[4] = pl.bx;
    q[5] = pl.by;
    const b200pt_render_node& rn = o.nodes[pl.rnodeID];
    const HitState hit = getHitState(o.prims[pl.rprimID], f3(1.0f - pl.bx - pl.by, pl.bx, pl.by), *(const mat4*)rn.worldToObject,
                                     *(const mat4*)rn.objectToWorld, (uint32_t)pl.primitiveID, r.d);
    const float    worldFoot = (p[9] + p[10] * pl.hitT) / fmaxf(fabsf(dot(hit.geonrm, -r.d)), 1e-3f);
    MeshState      mesh;
    mesh.N = hit.nrm;
    mesh.T = hit.tangent;
    mesh.B = hit.bitangent;
    mesh.Ng = hit.geonrm;
    mesh.tc[0] = hit.uv[0];
    mesh.tc[1] = hit.uv[1];
    mesh.isInside = p[8] != 0.0f;
    mesh.texGrad = worldFoot * hit.texelDensity * p[11];
    mesh.baseColorVertexMul = hit.color;
    const PbrMaterial m = evaluateMaterial(o, o.mats[std::max(0, rn.materialID)], mesh);
    putShadeField(q, 6, hit.pos);
    putShadeField(q, 9, hit.nrm);
    q[12] = hit.color.x;
    q[13] = hit.color.y;
    q[14] = hit.color.z;
    q[15] = hit.color.w;
    putShadeField(q, 16, hit.geonrm);
    putShadeField(q, 19, hit.shadowPos);
    q[22] = hit.uv[0].x;
    q[23] = hit.uv[0].y;
    q[24] = hit.uv[1].x;
    q[25] = hit.uv[1].y;
    putShadeField(q, 26, hit.tangent);
    putShadeField(q, 29, hit.bitangent);
    q[32] = hit.texelDensity;
    q[33] = mesh.texGrad;
    putShadeField(q, 34, m.baseColor);
    q[37] = m.opacity;
    q[38] = m.roughness.x;
    q[39] = m.roughness.y;
    q[40] = m.metallic;
    putShadeField(q, 41, m.emissive);
    putShadeField(q, 44, m.N);
    putShadeField(q, 47, m.T);
    putShadeField(q, 50, m.B);
    putShadeField(q, 53, m.Ng);
    q[56] = m.ior1;
    q[57] = m.ior2;
    q[58] = m.specular;
    putShadeField(q, 59, m.specularColor);
    q[62] = m.transmission;
    putShadeField(q, 63, m.attenuationColor);
    q[66] = m.attenuationDistance;
    q[67] = m.thickness;
    q[68] = m.clearcoat;
    q[69] = m.clearcoatRoughness;
    putShadeField(q, 70, m.Nc);
    q[73] = m.iridescence;
    q[74] = m.iridescenceIor;
    q[75] = m.iridescenceThickness;
    putShadeField(q, 76, m.sheenColor);
    q[79] = m.sheenRoughness;
    q[80] = m.dispersion;
    q[81] = m.diffuseTransmissionFactor;
    putShadeField(q, 82, m.diffuseTransmissionColor);
    putShadeField(q, 85, m.scatterCoefficient);
    q[88] = m.scatterAnisotropy;
    q[89] = m.retroreflection;
  }
  o.stats.merge();
  return 0;
}
}
