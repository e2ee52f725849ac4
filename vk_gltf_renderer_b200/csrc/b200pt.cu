// b200pt.cu — wavefront path-tracer kernels for sm_90a (H100) + the C-ABI of include/b200pt.h.
//
// Stage map (reference function -> kernel), SURVEY.md Appendix C:
//   processPixel head / samplePixel / getRay      gltf_pathtrace.slang:546-581,502-530  -> k_raygen (+ regen in finalizeSample)
//   IRaytracer::Trace: tree walks                  raytracer_interface.h.slang:69-122    -> k_trace (persistent warps)
//                      any-hit alpha tests         raytracer_interface.h.slang:82-112    -> k_alpha<false> (dense)
//   pathTraceOneBounce                             gltf_pathtrace.slang:87-430           -> k_shade
//   IRaytracer::TraceShadow: tree walks            raytracer_interface.h.slang:139-187   -> k_shadow (persistent warps)
//                      any-hit transmission        raytracer_interface.h.slang:149-179   -> k_alpha<true> (dense)
//   NEE add + RR + depth++ (pathTrace tail)        gltf_pathtrace.slang:462-485          -> k_resolve
//   accumulation                                   gltf_pathtrace.slang:582-630          -> k_accumulate
//   shadow catcher (handleShadowCatcher)           pathtrace_functions.h.slang:499-554   -> k_shade (light sample) + shadow kernels + finishPost
//   eOptixAlbedoNormal guide image                 gltf_pathtrace.slang:240-263,653-670  -> capture in k_shade, k_guide
//   DLSS variant: jitter, guides, motion vectors   gltf_pathtrace.slang:135-143,216-263,370-377,564-651 -> k_raygen, k_shade, k_dlss_guides
//   snapshot_prev_transforms.comp                  src/renderer.cpp:630-655                               -> k_snapshot_prev_transforms
// Next to the frame path (SURVEY.md section 8 f):
//   morph.comp / skinning.comp                     shaders/*.comp.slang                  -> k_morph, k_skin, k_regather_shade (animate.cuh)
//   world_matrix_propagate / update_render_instances                                     -> k_propagate_level, k_update_render_nodes
//   BLAS / TLAS build and update                   src/gltf_scene_rtx.cpp:173-503        -> k_lbvh_* (lbvh.cuh), k_refit_* (refit.cuh)
//   updateSceneChanges: material edits             src/renderer.cpp:2269-2362            -> k_retag_tris, k_gather_alpha (or a tree rebuild)
//   GltfRenderer::tonemap                          src/renderer.cpp:992-1054             -> k_tm_histogram, k_tm_exposure, k_tonemap (tonemap.cuh)
// One path slot per pixel; samples of a pixel within a frame run back to back in the same slot
// (path regeneration) because the reference continues ONE rng stream across a pixel's samples.
#include <cuda_runtime.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "bvh.h"
#include "animate.cuh"
#include "dlss_guides.cuh"
#include "lbvh.cuh"
#include "shade.cuh"
#include "tonemap.cuh"

using namespace pt;

static_assert(sizeof(b200pt_render_node) == 136, "GltfRenderNode layout");
static_assert(sizeof(b200pt_texture_info) == 32, "GltfTextureInfo layout");
static_assert(sizeof(b200pt_shade_material) == 288, "GltfShadeMaterial layout");
static_assert(sizeof(b200pt_light) == 64, "GltfLight layout");
static_assert(sizeof(b200pt_frame_info) == 396, "SceneFrameInfo layout");
static_assert(sizeof(b200pt_push_constant) == 48, "PathtracePushConstant layout");

namespace {

constexpr int kMaxIters = 4096;  // per-frame iteration counter slots
// the six DLSS guide planes of one pixel: albedo RGBA8 (4 B), specular albedo RGBA16F (8), normal / roughness RGBA16F (8),
// motion RG16F (4), depth R16F (2), specular hit distance R16F (2)
constexpr size_t kDlssBytesPerPixel = 28;
// Any-hit continuation rounds per bounce: a ray whose kCand candidates were all rejected goes through another k_trace / k_shadow round
// that resumes behind the last one; after kContRoundsMax rounds whatever is still undecided finishes inside the last k_alpha.
constexpr int kContRoundsMax = 8;

// The per-iteration device counters (queue sizes, dynamic-fetch cursors of the persistent walks): kArrays arrays of `stride` words, word
// `it` of each for iteration `it` (a frame: kMaxIters bounces; the ray-level API: one).  Per ray kind (0 closest, 1 shadow): the walk's
// cursor, the any-hit counters of round r (r = 0: the main walk's candidates), the continuation counters and cursors of round r.
struct Counters
{
  uint32_t* base;
  size_t    stride;
  static constexpr int kPerKind = 3 * kContRoundsMax + 1;
  static constexpr int kArrays = 5 + 2 * kPerKind;
  uint32_t* at(int array, int it) const { return base + (size_t)array * stride + (size_t)it; }
  uint32_t* trace(int it) const { return at(0, it); }   // closest-hit rays (k_raygen / k_shade / k_resolve append, k_trace reads)
  uint32_t* post(int it) const { return at(1, it); }    // paths for k_resolve
  uint32_t* shadow(int it) const { return at(4, it); }  // shadow rays
  uint32_t* queue(int kind, int it) const { return kind ? shadow(it) : trace(it); }  // the rays a walk of this kind reads
  uint32_t* cursor(int kind, int it) const { return at(2 + kind, it); }
  uint32_t* anyHit(int kind, int r, int it) const { return at(5 + kind * kPerKind + r, it); }
  uint32_t* cont(int kind, int r, int it) const { return at(5 + kind * kPerKind + kContRoundsMax + 1 + r, it); }
  uint32_t* contCursor(int kind, int r, int it) const { return at(5 + kind * kPerKind + 2 * kContRoundsMax + 1 + r, it); }
};
constexpr int kCounterArrays = Counters::kArrays;

// stages of the profiling events: the per-stage times and launch counts of b200pt_stats and the stage column of a B200PT_TIMELINE dump
enum Stage : int
{
  kStageTrace = 0,  // closest-hit walks
  kStageShade = 1,
  kStageShadow = 2,  // shadow walks
  kStageOther = 3,
  kStageAnyHit = 4,
  kStageResolve = 5,
  kStageCount
};
constexpr const char* kStageName[kStageCount] = {"k_trace", "k_shade", "k_shadow", "other", "k_alpha", "k_resolve"};

// -------------------------------------------------------------------------------------------------
// queue helper: warp-aggregated append
// -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void queuePush(uint32_t* q, uint32_t* cnt, uint32_t value)
{
  const unsigned mask = __activemask();
  const int      lane = threadIdx.x & 31;
  const int      leader = __ffs(mask) - 1;
  uint32_t       base = 0;
  if(lane == leader)
    base = atomicAdd(cnt, (uint32_t)__popc(mask));
  base = __shfl_sync(mask, base, leader);
  q[base + __popc(mask & ((1u << lane) - 1u))] = value;
}

__device__ __forceinline__ void statAdd(unsigned long long* p, unsigned long long v)
{
  // per-warp aggregation of a uniform +v
  const unsigned mask = __activemask();
  const int      lane = threadIdx.x & 31;
  if(lane == __ffs(mask) - 1)
    atomicAdd(p, v * (unsigned long long)__popc(mask));
}

// -------------------------------------------------------------------------------------------------
// camera ray + sample start (samplePixel head: gltf_pathtrace.slang:502-530; getRay: pathtrace_functions.h.slang:791-811)
// -------------------------------------------------------------------------------------------------
// the pinhole or orthographic camera ray through pixel (x, y) + offset
__device__ __forceinline__ void getRay(const FrameParams& F, const Camera& cam, uint32_t x, uint32_t y, float2 offset, float3& org, float3& dir)
{
  const Mat4&  projI = *reinterpret_cast<const Mat4*>(F.fi.projInv);
  const Mat4&  viewI = *reinterpret_cast<const Mat4*>(cam.viewInv);
  const float2 clip = f2(((float)x + offset.x) / F.fi.imageSize[0] * 2.0f - 1.0f, ((float)y + offset.y) / F.fi.imageSize[1] * 2.0f - 1.0f);
  float4       vc = mul_vM(f4(clip.x, clip.y, -1.0f, 1.0f), projI);
  vc = vc / vc.w;
  if(F.fi.flags & B200PT_SCENE_IS_ORTHOGRAPHIC)
  {
    org = xyz(mul_vM(vc, viewI));
    dir = normalize(xyz(mul_vM(f4(0, 0, -1, 0), viewI)));
  }
  else
  {
    org = f3(viewI.m[12], viewI.m[13], viewI.m[14]);
    dir = normalize(xyz(mul_vM(vc, viewI)) - org);
  }
}

__device__ void startSample(const PathState& P, const FrameParams& F, uint32_t i, uint32_t seed, float2 jitter, uint32_t sampleIdx)
{
  const uint32_t px = pixelOf(F, i);
  const Camera   cam = cameraOf(F, i);
  float3         org, dir;
  getRay(F, cam, px % (uint32_t)F.width, pixelRow(F, px), jitter, org, dir);
  if(!(F.fi.flags & B200PT_SCENE_IS_ORTHOGRAPHIC))
  {
    const Mat4& viewI = *reinterpret_cast<const Mat4*>(cam.viewInv);
    // thin-lens DOF: the two rand() are consumed even when aperture == 0 (:519-520)
    const float3 focalPoint = dir * F.pc.focalDistance;
    const float  cam_r1 = rnd(seed) * kTwoPi;
    const float  cam_r2 = rnd(seed) * F.pc.aperture;
    const float4 camRight = mul_Mv(viewI, f4(1, 0, 0, 0));
    const float4 camUp = mul_Mv(viewI, f4(0, 1, 0, 0));
    const float3 rap = (xyz(camRight) * cosf(cam_r1) + xyz(camUp) * sinf(cam_r1)) * sqrtf(cam_r2);
    dir = normalize(focalPoint - rap);
    org += rap;
  }
  dir = normalize(dir);  // pathTrace() re-normalises at the top of every loop iteration (:447)
  P.rayO[i] = f4(org, 0.0f);
  P.rayD[i] = f4(dir, kInfinite);
  P.thr[i] = f4(1.0f, 1.0f, 1.0f, kDirac);
  P.rad[i] = f4(0.0f, 0.0f, 0.0f, __uint_as_float(0u));
  P.misc[i] = f4(0.0f, 0.0f, __uint_as_float(PF_SOLID), __uint_as_float(seed));
  P.medium[i] = make_uint4(0u, 0u, 0u, sampleIdx << 16);
  if(isFirstFrame(F, i))
    P.firstHit[i] = f4(1e34f, 1e34f, 1e34f, 1.0f);  // PathTracerState::firstHitPos sentinel, pt.solid = true
  if(P.guideA)
  {
    P.guideA[i] = f4(0.f, 0.f, 0.f, 0.f);  // GuideScratch defaults: albedo 0, normalRoughness 0
    P.guideN[i] = f4(0.f, 0.f, 0.f, 0.f);
  }
}

// end of one samplePixel(): firefly clamp, add to the pixel sum, start the pixel's next sample if any
__device__ void finalizeSample(const PathState& P, const FrameParams& F, uint32_t i, float3 radiance, bool solid, uint32_t seed, uint32_t sampleIdx,
                               uint32_t* qNext, uint32_t* cntNext, DevStats* stats)
{
  float4      r = f4(radiance, solid ? 1.0f : 0.0f);
  const float lum = (r.x + r.y + r.z) * (1.0f / 3.0f);
  if(lum > F.pc.fireflyClampThreshold)
    r = r * (F.pc.fireflyClampThreshold / lum);
  P.pixSum[i] = P.pixSum[i] + r;
  const uint32_t s = sampleIdx + 1;
  if((int)s < F.pc.numSamples)
  {
    const float a = rnd(seed), b = rnd(seed);
    startSample(P, F, i, seed, f2(a, b), s);
    statAdd(&stats->pathsStarted, 1ull);
    queuePush(qNext, cntNext, i);
  }
}

// -------------------------------------------------------------------------------------------------
// kernels
// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_raygen(PathState P, const __grid_constant__ FrameParams F, uint32_t* qTrace, uint32_t* cnt0, DevStats* stats)
{
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < F.numPaths; i += stride)
  {
    const uint32_t px = pixelOf(F, i);
    const uint32_t x = px % (uint32_t)F.width;
    const uint32_t y = pixelRow(F, px);
    uint32_t       seed = xxhash32(x, y, (uint32_t)F.pc.frameCount + frameOf(F, i));
    uint32_t       drawn = seed;
    const float    u1 = rnd(drawn), u2 = rnd(drawn);
    // sampleGaussian (pathtrace_functions.h.slang:784-789), sigma = 0.4246609 px
    const float    rr = sqrtf(-2.0f * logf(fmaxf(1e-38f, u1)));
    const float    theta = 2.0f * kPi * u2;
    float2         jitter = f2(0.5f + (rr * cosf(theta)) * 0.4246609f, 0.5f + (rr * sinf(theta)) * 0.4246609f);
    // the DLSS jitter moves the whole frame and the Gaussian's two rand() are not drawn (gltf_pathtrace.slang:568-572)
    if(F.pc.flags & B200PT_PT_USE_DLSS)
      jitter = f2(0.5f + F.fi.jitter[0], 0.5f + F.fi.jitter[1]);
    else
      seed = drawn;
    P.pixSum[i] = f4(0.f, 0.f, 0.f, 0.f);
    if(isDlssFrame(P, F))
    {
      // a DLSS frame has one sample, started here: the first-hit scratch of every frame and the DLSS GuideScratch defaults
      P.firstHit[i] = f4(1e34f, 1e34f, 1e34f, 1.0f);
      P.prevHit[i] = f4(1e34f, 1e34f, 1e34f, 1.0f);  // firstHitPosPrev sentinel
      P.dlssSpec[i] = make_uint2(0u, 0u);            // specularAlbedo 0, specularHitDist 0
    }
    startSample(P, F, i, seed, jitter, 0u);
    qTrace[i] = i;
  }
  if(blockIdx.x == 0 && threadIdx.x == 0)
  {
    *cnt0 = F.numPaths;
    atomicAdd(&stats->pathsStarted, (unsigned long long)F.numPaths);
  }
}

// Persistent-warp scheme (Aila & Laine 2009 style): all 32 lanes of a warp reconverge at the fetch point
// (__syncwarp), lanes that finished their ray take the next queue entries from a global cursor, then the
// warp walks the tree until fewer than kRefillThreshold lanes are still busy and goes back to refill.
constexpr int kRefillThreshold = 22;
// 64 registers: 8 walk CTAs of 128 threads per SM (the 64 K-register file of an H100 SM full); also the walks' persistent grid
constexpr int kWalkCtasPerSM = 8;
// threads per walk CTA, also the column stride of the walks' shared candidate lists
constexpr int kWalkBlock = 128;

// full-warp fetch: every lane calls it; lanes with need==true receive the next queue slot or 0xFFFFFFFF
__device__ __forceinline__ uint32_t fetchWork(bool need, uint32_t* workCounter, uint32_t count)
{
  const unsigned want = __ballot_sync(0xffffffffu, need);
  if(want == 0)
    return 0xFFFFFFFFu;
  const int lane = threadIdx.x & 31;
  const int leader = __ffs(want) - 1;
  uint32_t  base = 0;
  if(lane == leader)
    base = atomicAdd(workCounter, (uint32_t)__popc(want));
  base = __shfl_sync(0xffffffffu, base, leader);
  if(!need)
    return 0xFFFFFFFFu;
  const uint32_t k = base + (uint32_t)__popc(want & ((1u << lane) - 1u));
  return k < count ? k : 0xFFFFFFFFu;
}

// The persistent-warp loop of the walk kernels, over the `count` paths of queue q.  Per lane: path (-1 needs work, -2
// exhausted) and a resumable traversal; finished lanes are handled in the converged part of the loop, never inside the
// traversal loop.  start(T, path) begins the walk of a fetched path; finish(T, cand, path) writes a finished walk out and
// returns whether the lane is free (false: it started T again on the same path).  OMM, CAPS, MODE and omm are those of
// TravState::step (MODE 1: closest-hit walk, 2: shadow walk); a continuation round (cont) does not count its rays again.
template <bool OMM, bool CAPS, int MODE, class Start, class Finish>
__device__ __forceinline__ void walkQueue(const uint32_t* __restrict__ q, uint32_t count, uint32_t* workCounter, const BvhView& omm, DevStats* stats, bool cont,
                                          Start start, Finish finish)
{
  __shared__ Cand s_cand[kCand * kWalkBlock];  // candidate lists, one column per thread (20-byte stride: conflict-free)
  Cand* const     cand = &s_cand[threadIdx.x];
  TravState       T;
  uint2           stack[TravState::kStackSize];
  int             path = -1;
  bool            travDone = false;  // traversal finished, write-out pending
  for(;;)
  {
    __syncwarp();
    if(path >= 0 && travDone)
    {
      travDone = false;
      T.flushCounters(&stats->nodesVisited, &stats->trisTested);
      const bool overflow = T.overflow;  // (finish may start T again)
      if(finish(T, cand, path))
        path = -1;
      if(overflow)
        atomicOr(&stats->errorFlags, 1ull);
    }
    __syncwarp();
    // ---- refill ----
    {
      const bool     need = (path == -1);
      const uint32_t k = fetchWork(need, workCounter, count);
      if(need)
      {
        if(k == 0xFFFFFFFFu)
          path = -2;
        else
        {
          path = (int)q[k];
          start(T, path);
        }
      }
    }
    if(__all_sync(0xffffffffu, path == -2))
      break;
    // ---- traverse: warp-uniform loop (all 32 lanes iterate, idle lanes are predicated off) until too few
    //      lanes are still busy ----
    for(;;)
    {
#ifdef B200PT_COUNT_TRAVERSAL
      {
        const unsigned busy = __ballot_sync(0xffffffffu, path >= 0 && !travDone);
        if((threadIdx.x & 31) == 0)
        {
          atomicAdd(&stats->warpIters, 1ull);
          atomicAdd(&stats->busyLaneIters, (unsigned long long)__popc(busy));
        }
      }
#endif
      if(path >= 0 && !travDone)
        travDone = T.step<kCand, false, OMM, MODE, CAPS>(stack, kPostponeShift, cand, kWalkBlock, omm.ommRef, omm.ommData, omm.capRef, omm.capBits);
      if(__popc(__ballot_sync(0xffffffffu, path >= 0 && !travDone)) < kRefillThreshold)
        break;
    }
  }
  if(blockIdx.x == 0 && threadIdx.x == 0 && !cont)
    atomicAdd(MODE == 1 ? &stats->closestRays : &stats->shadowRays, (unsigned long long)count);
}

// is every one of the n candidates a cap or a hole (tagged by the CAPS walk)?
__device__ __forceinline__ bool knownOpacities(const Cand* cand, int n)
{
  bool known = true;
#pragma unroll
  for(int i = 0; i < kCand; i++)
    if(i < n)
      known &= (cand[i * kWalkBlock].slot & (kCandCap | kCandHole)) != 0;
  return known;
}
// the first n candidates into the path state for k_alpha (a CAPS walk's tags cleared)
template <bool CAPS>
__device__ __forceinline__ void writeCandidates(const PathState& P, uint32_t path, const Cand* cand, int n)
{
#pragma unroll
  for(int i = 0; i < kCand; i++)
    if(i < n)
    {
      const Cand c = cand[i * kWalkBlock];
      P.cand[i][path] = f4(c.t, c.u, c.v, __uint_as_float(CAPS ? c.slot & kCandSlot : c.slot));
    }
}

// IRaytracer::Trace, geometry part, for every path in the queue: ONE walk of the scene tree gives the closest
// FORCE_OPAQUE hit and the kCand nearest any-hit candidates in front of it (traverse.cuh).  The stochastic alpha
// tests need textures and touch only the few lanes whose walk just ended -- inside this kernel they ran with ~2 of
// 32 lanes active and took a large share of its instructions and stall samples -- so they live in
// the dense kernel k_alpha; this kernel only writes the candidates out.
// mode: TRACE_CONT = continuation round (the paths in the queue had all kCand candidates rejected by k_alpha and resume
// behind the last one; P.hit seeds the opaque bound and is refined), TRACE_TMIN = rayO.w carries tmin (ray-level API).
enum : int
{
  TRACE_CONT = 1,
  TRACE_TMIN = 2,
};
template <bool OMM, bool CAPS>
__global__ void __launch_bounds__(kWalkBlock, kWalkCtasPerSM) k_trace(PathState P, DevScene S, const uint32_t* __restrict__ q, const uint32_t* __restrict__ cntIn,
                                                                      uint32_t* workCounter, uint32_t* qAlpha, uint32_t* cntAlpha, DevStats* stats, int mode)
{
  const bool cont = (mode & TRACE_CONT) != 0;
  auto       start = [&](TravState& T, int path) {
    const float4 o = P.rayO[path];
    const float4 d = P.rayD[path];
    const float  tmin = (mode & TRACE_TMIN) ? o.w : 0.0f;
    if(!cont)
      T.init(S.bvh, xyz(o), xyz(d), tmin, d.w, true, false, false, 0.f, 0u);
    else
    {
      T.init(S.bvh, xyz(o), xyz(d), tmin, d.w, true, false, true, P.cand[kCand - 1][path].x, P.candInfo[path].y);
      const float4 hp = P.hit[path];
      if(__float_as_uint(hp.w) != 0xFFFFFFFFu)
        T.seedOpaque(hp.x, hp.y, hp.z, __float_as_uint(hp.w));
    }
  };
  auto finish = [&](TravState& T, const Cand* cand, int path) {
    const TraceHit ho = T.result();
    P.hit[path] = f4(ho.t, ho.u, ho.v, __uint_as_float(ho.slot));
    const int n = T.candidatesInFront(cand, kWalkBlock);
    if(n > 0)
    {
      // every candidate a cap or a hole (alpha_caps.cuh): its opacity is exactly 1 or 0, so the draws alone decide the any-hit loop of
      // k_alpha<false> and it runs here, without texels -- unless all kCand were rejected and a continuation round must follow
      if(CAPS && knownOpacities(cand, n))
      {
        uint32_t* const seedOut = reinterpret_cast<uint32_t*>(&P.misc[path]) + 3;
        uint32_t        seed = *seedOut;
        int             acc = -1;
#pragma unroll
        for(int i = 0; i < kCand; i++)
          if(i < n && acc < 0 && rnd(seed) <= ((cand[i * kWalkBlock].slot & kCandCap) ? 1.0f : 0.0f))
            acc = i;
        if(acc >= 0 || n < kCand)
        {
          if(acc >= 0)
          {
            const Cand     c = cand[acc * kWalkBlock];
            const uint32_t slot = c.slot & kCandSlot;
            const bool     flip = ((__float_as_uint(__ldg(&S.bvh.tris[slot * 3 + 0]).w) >> 28) & TRI_FLIPPED) != 0;
            P.hit[path] = f4(c.t, flip ? c.v : c.u, flip ? c.u : c.v, __uint_as_float(slot));
          }
          *seedOut = seed;
          return true;
        }
      }
      writeCandidates<CAPS>(P, path, cand, n);
      P.candInfo[path] = make_uint2((uint32_t)n, cand[(n - 1) * kWalkBlock].gid);
      queuePush(qAlpha, cntAlpha, (uint32_t)path);
    }
    return true;
  };
  walkQueue<OMM, CAPS, 1>(q, *cntIn, workCounter, S.bvh, stats, cont, start, finish);
}

// Any-hit part of IRaytracer::Trace (SHADOW = false) and IRaytracer::TraceShadow (SHADOW = true): the candidates
// the geometry kernel collected, nearest first, one rand() each (raytracer_interface.h.slang:82-112, 149-179, with
// the order pinned to (t, triangle id)).
//   Trace:       the first candidate that passes its alpha test replaces the opaque hit.
//   TraceShadow: every candidate that passes multiplies the transmission (0 for MASK / opaque-ish materials);
//                the result is folded into the path's pending NEE contribution.
// kCand lanes per path: lane j evaluates the opacity of candidate j (the texture fetches -- the long latency chain
// -- run in parallel), then all of them replay the same sequential decisions and lane 0 writes.  A path whose
// kCand candidates are used up goes to the continuation queue (another k_trace / k_shadow round resumes the walk
// behind the last candidate); in the last round (qCont == nullptr) it keeps walking right here instead.
template <bool SHADOW>
__global__ void __launch_bounds__(128) k_alpha(PathState P, DevScene S, const uint32_t* __restrict__ q, const uint32_t* __restrict__ cntIn, uint32_t* qCont,
                                               uint32_t* cntCont, DevStats* stats, int mode)
{
  static_assert(kCand == 2 || kCand == 4 || kCand == 8, "kCand lanes per path");
  // candidate slots index the triangle array of the tree that produced them: the merged tree for closest-hit rays,
  // the split opaque / non-opaque arrays for shadow rays
  const uint2* __restrict__ triMeta = SHADOW ? S.triMetaS : S.triMeta;
  constexpr int             KF = 16;  // candidates per walk of the in-kernel fallback (its list lives in local memory)
  // the opacity of a candidate of the fallback walks, and its (u, v) with a mirrored instance's swap undone
  auto fallbackOpacity = [&](const Cand& c, float& u, float& v) {
    const uint2               meta = triMeta[c.slot];
    const bool                flip = ((meta.x >> 28) & TRI_FLIPPED) != 0;
    u = flip ? c.v : c.u;
    v = flip ? c.u : c.v;
    const b200pt_render_node& node = S.nodes[meta.x & 0x0fffffffu];
    return getOpacity(S, node, S.prims[node.renderPrimID], meta.y, f3(1.0f - u - v, u, v));
  };
  stageSrgbLut(S.lutSrgb);
  const uint32_t count = *cntIn;
  constexpr int  G = kCand, PPW = 32 / kCand;  // lanes per path, paths per warp
  const int      lane = threadIdx.x & 31, sub = lane % G, grp = lane / G, base = lane - sub;
  const uint32_t warpsTotal = gridDim.x * (blockDim.x >> 5);
  const uint32_t warpId = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  for(uint32_t k0 = warpId * (uint32_t)PPW; k0 < count; k0 += warpsTotal * (uint32_t)PPW)  // warp-uniform trip count
  {
    const uint32_t k = k0 + (uint32_t)grp;
    const bool     valid = k < count;
    uint32_t       path = 0;
    uint2          info = make_uint2(0u, 0u);
    if(valid)
    {
      path = q[k];
      info = P.candInfo[path];
    }
    const int n = (int)(info.x & 0xffu);
    // ---- lane j: candidate j and its opacity ----
    float    ct = 0.f, cu = 0.f, cv = 0.f, op = 0.f, transmission = 0.f;
    uint32_t slot = 0;
    if(sub < n)
    {
      const float4 c = P.cand[sub][path];
      slot = __float_as_uint(c.w);
      // the triangle's pre-gathered alpha record: candidate -> (index ->) record -> texels
      const uint32_t ri = SHADOW ? slot - S.alphaBaseS : __ldg(&S.alphaIdx[slot]);
      const uint32_t w0 = __float_as_uint(__ldg(&(SHADOW ? S.bvhA.tris : S.bvh.tris)[slot * 3 + 0]).w);
      const bool     flip = ((w0 >> 28) & TRI_FLIPPED) != 0;  // mirrored instance: (u, v) swap back
      const AlphaRec rec = loadAlphaRec(S.alphaRecs + ri);
      ct = c.x;
      cu = flip ? c.z : c.y;
      cv = flip ? c.y : c.z;
      op = opacityFromRecord(rec, f3(1.0f - cu - cv, cu, cv));
      transmission = rec.transmission;
    }
    const uint32_t seedIn = valid ? __float_as_uint(P.misc[path].w) : 0u;
    uint32_t       seed = seedIn;
    if(!SHADOW)
    {
      int acc = -1;
#pragma unroll
      for(int i = 0; i < kCand; i++)
      {
        const float oi = __shfl_sync(0xffffffffu, op, base + i);
        if(i < n && acc < 0 && rnd(seed) <= oi)
          acc = i;
      }
      if(acc >= 0 && sub == acc)
        P.hit[path] = f4(ct, cu, cv, __uint_as_float(slot));
      const float    lastT = __shfl_sync(0xffffffffu, ct, base + kCand - 1);
      if(acc < 0 && n == kCand && qCont != nullptr)
      {
        if(sub == 0)
          queuePush(qCont, cntCont, path);
      }
      else if(acc < 0 && n == kCand)
      {
        // every collected candidate was rejected and there may be more: keep walking, kCand at a time (the lanes of
        // the group do this redundantly, lane 0 writes).  Each walk also refines the opaque hit (traverse.cuh).
        const float4 o = P.rayO[path], d = P.rayD[path], hp = P.hit[path];
        const float  tmin = (mode & TRACE_TMIN) ? o.w : 0.0f;
        TraceHit     opq;
        opq.slot = 0xFFFFFFFFu;
        if(__float_as_uint(hp.w) != 0xFFFFFFFFu)
          opq = seedHit(S.bvh, hp.x, hp.y, hp.z, __float_as_uint(hp.w));
        float    loT = lastT;
        uint32_t loId = info.y;
        Cand     cand[KF];
        bool     accepted = false, overflowed = false;
        for(;;)
        {
          const int m = walkCollect<KF>(S.bvh, xyz(o), xyz(d), tmin, d.w, true, false, true, true, loT, loId, opq, cand, &overflowed);
          for(int i = 0; i < m && !accepted; i++)
          {
            float       u, v;
            const float opacity = fallbackOpacity(cand[i], u, v);
            if(rnd(seed) <= opacity)
            {
              if(sub == 0)
                P.hit[path] = f4(cand[i].t, u, v, __uint_as_float(cand[i].slot));
              accepted = true;
            }
          }
          if(accepted || m < KF)
            break;
          loT = cand[KF - 1].t;
          loId = cand[KF - 1].gid;
        }
        if(!accepted && sub == 0 && opq.slot != 0xFFFFFFFFu)
        {
          const TraceHit ho = unflipHit(opq);
          P.hit[path] = f4(ho.t, ho.u, ho.v, __uint_as_float(ho.slot));
        }
        if(overflowed && sub == 0)
          atomicOr(&stats->errorFlags, 1ull);
      }
    }
    else
    {
      // a continuation round resumes with the running transmission and segment start the previous round parked
      // in P.hit (free between shading and the next k_trace)
      const float4 saved = (valid && (mode & TRACE_CONT)) ? P.hit[path] : f4(1.0f, 1.0f, 1.0f, 0.0f);
      float3       total = xyz(saved);
      float        prevHitT = saved.w;
      bool         done = false, parked = false;
      const float4 misc = valid ? P.misc[path] : f4(0, 0, 0, 0);
      bool         isInside = (__float_as_uint(misc.z) & PF_SHADOW_INSIDE) != 0;
      const float3 dir = valid ? xyz(P.shD[path]) : f3(0, 0, 1);
      auto         accept = [&](uint32_t sl, float t, float u, float v) {
        const uint2               meta = triMeta[sl];
        const b200pt_render_node& node = S.nodes[meta.x & 0x0fffffffu];
        const float               seg = fmaxf(0.0f, t - prevHitT);
        const float3              cur = getShadowTransmission(S, node, S.prims[node.renderPrimID], meta.y, f3(1.0f - u - v, u, v), seg, dir, isInside);
        prevHitT = t;
        total *= cur;
        if(maxc(total) <= 0.01f)
        {
          total = f3(0.0f);
          done = true;
        }
      };
#pragma unroll
      for(int i = 0; i < kCand; i++)
      {
        const float    oi = __shfl_sync(0xffffffffu, op, base + i);
        const float    ti = __shfl_sync(0xffffffffu, ct, base + i);
        const float    ui = __shfl_sync(0xffffffffu, cu, base + i);
        const float    vi = __shfl_sync(0xffffffffu, cv, base + i);
        const uint32_t si = __shfl_sync(0xffffffffu, slot, base + i);
        const float    tr = __shfl_sync(0xffffffffu, transmission, base + i);
        if(i < n && !done && rnd(seed) < oi)
        {
          if(tr <= 0.01f)
          {
            // getShadowTransmission returns 0 for a non-transmissive material (alpha-tested foliage): the ray is blocked
            // (same result as accept(), without its gathers)
            prevHitT = ti;
            total = f3(0.0f);
            done = true;
          }
          else
            accept(si, ti, ui, vi);
        }
      }
      const float lastT = __shfl_sync(0xffffffffu, ct, base + kCand - 1);
      if(!done && n == kCand && qCont != nullptr)
      {
        parked = true;
        if(sub == 0)
        {
          P.hit[path] = f4(total, prevHitT);
          const uint32_t fl = (__float_as_uint(misc.z) & ~PF_SHADOW_INSIDE) | (isInside ? PF_SHADOW_INSIDE : 0u);
          reinterpret_cast<uint32_t*>(&P.misc[path])[2] = fl;
          queuePush(qCont, cntCont, path);
        }
      }
      else if(!done && n == kCand)
      {
        // more than kCand layers on the segment: keep walking, kCand at a time (rare)
        const float4 so = P.shO[path];
        float        loT = lastT;
        uint32_t     loId = info.y;
        Cand         cand[KF];
        bool         overflowed = false;
        while(!done)
        {
          TraceHit opq;
          opq.slot = 0xFFFFFFFFu;
          const int m = walkCollect<KF>(S.bvhA, xyz(so), dir, 0.0f, so.w, false, true, true, true, loT, loId, opq, cand, &overflowed);
          if(opq.slot != 0xFFFFFFFFu)
          {
            // (the first walk of the segment found no opaque occluder, so none can turn up here)
            total = f3(0.0f);
            done = true;
          }
          for(int i = 0; i < m && !done; i++)
          {
            float       u, v;
            const float opacity = fallbackOpacity(cand[i], u, v);
            if(rnd(seed) < opacity)
              accept(cand[i].slot, cand[i].t, u, v);
          }
          if(m < KF)
            break;
          loT = cand[KF - 1].t;
          loId = cand[KF - 1].gid;
        }
        if(overflowed && sub == 0)
          atomicOr(&stats->errorFlags, 1ull);
      }
      if(valid && sub == 0 && !parked)
      {
        const float4 c = P.shC[path];
        P.shC[path] = f4(xyz(c) * total, c.w);
      }
    }
    if(valid && sub == 0 && seed != seedIn)
      reinterpret_cast<uint32_t*>(&P.misc[path])[3] = seed;
  }
}

// the infinite plane's material, gltf_pathtrace.slang:169-173: defaultPbrMaterial(infinitePlaneBaseColor, metallic, roughness, N, N)
// (nvshaders, external: restated -- GGX alpha = roughness^2 like evaluateMaterial, tangent frame from the normal; same in the oracle)
__device__ __forceinline__ PbrMaterial planeMaterial(const FrameParams& F)
{
  const float3 n = f3(0, 1, 0);
  PbrMaterial  m = defaultPbrMaterial();
  m.baseColor = f3(F.fi.infinitePlaneBaseColor[0], F.fi.infinitePlaneBaseColor[1], F.fi.infinitePlaneBaseColor[2]);
  m.metallic = F.fi.infinitePlaneMetallic;
  const float r = F.fi.infinitePlaneRoughness;
  m.roughness = f2(r * r, r * r);
  m.N = m.Ng = m.Nc = n;
  m.T = xyz(makeFastTangent(n));
  m.B = cross(m.N, m.T);
  return m;
}

// H100 (SynthSponza 1080p bench): 256-thread CTAs at <= 255 registers run without spills and beat 512 at <= 128
constexpr int kShadeBlock = 256;
constexpr int kShadeCtasPerSM = 2;  // CTAs per SM of the persistent shade grid
template <uint32_t FEAT>
__global__ void __launch_bounds__(kShadeBlock, 1) k_shade(PathState P, DevScene S, const __grid_constant__ FrameParams F, const uint32_t* __restrict__ q,
                                                          const uint32_t* __restrict__ cntIn, uint32_t* qPost, uint32_t* cntPost, uint32_t* qShadow, uint32_t* cntShadow,
                                                          uint32_t* qNext, uint32_t* cntNext, DevStats* stats)
{
  stageSrgbLut(S.lutSrgb);
  const uint32_t count = *cntIn;
  const uint32_t stride = gridDim.x * blockDim.x;
  // One path per thread per pass.  The kernel is ~12 000 straight-line instructions that every warp walks once per
  // path, so it is bound by instruction fetch (ncu: no_instruction is its top stall, 20 % issue utilisation); the
  // block-uniform loop with a barrier per pass keeps the eight warps of a 256-thread block inside the same stretch of
  // code so they share the fetched lines.
  // pass state shared by the four sections of a pass (see the pass loop below)
  uint32_t                  i = 0, flags = 0, seed = 0, scatterBounces = 0, sampleIdx = 0, depth = 0, slot = 0;
  float4                    hr, misc;
  uint4                     med;
  float3                    org, dir, throughput, radiance;
  float                     coneWidth = 0.f, lastSamplePdf = 0.f, hitT = 0.f, worldFoot = 0.f;
  uint2                     meta;
  const b200pt_render_node* nodeP = nullptr;
  HitState                  hit;
  PbrMaterial               pbrMat;
  DirectLight               directLight;
  bool                      nextEventValid = false;
  bool                      onPlane = false;  // the ray met the infinite ground plane in front of the geometry
  bool                      catcher = false;  // ... and the plane is a shadow catcher (handleShadowCatcher, pathtrace_functions.h.slang:499-554)
#ifdef B200PT_DEBUG
  bool dbgPixel = false;
#endif
  // ---- section 1: path state, environment hit (path ends), hit attributes ----
  auto shadeLoad = [&](const uint32_t k) -> bool {
    i = q[k];
    const float4   ro = P.rayO[i];
    const float4   rd = P.rayD[i];
    hr = P.hit[i];
    float4         thr4 = P.thr[i];
    float4         rad4 = P.rad[i];
    misc = P.misc[i];
    med = P.medium[i];
    org = xyz(ro);
    dir = xyz(rd);
    coneWidth = ro.w;
    throughput = xyz(thr4);
    radiance = xyz(rad4);
    lastSamplePdf = thr4.w;
    flags = __float_as_uint(misc.z);
    seed = __float_as_uint(misc.w);
    scatterBounces = __float_as_uint(rad4.w);
    sampleIdx = med.w >> 16;
    depth = flags & PF_DEPTH_MASK;
    slot = __float_as_uint(hr.w);
    hitT = hr.x;

    // ---- infinite ground plane (checkInfinitePlaneIntersection, pathtrace_functions.h.slang:556-585): y = infinitePlaneDistance,
    //      hit from above only, when it lies in front of the geometry hit ----
    onPlane = false;
    catcher = false;
    if(F.fi.flags & B200PT_SCENE_USE_INFINITE_PLANE)
    {
      const float3 normal = f3(0, 1, 0);
      const float  planeHeight = F.fi.infinitePlaneDistance;
      const float  tGeom = (slot == 0xFFFFFFFFu) ? kInfinite : hitT;
      if(!(org.y <= planeHeight))
      {
        const float Dn = dot(dir, normal);
        if(!(fabsf(Dn) <= 1e-6f))
        {
          const float On = dot(org, normal);
          const float intersectionDist = (-On + planeHeight) / Dn;
          if(!(intersectionDist <= 0.0f || intersectionDist >= tGeom))
          {
            onPlane = true;
            hitT = intersectionDist;
            hit.pos = org + dir * hitT;
            hit.shadowPos = hit.pos;
            hit.nrm = normal;
            hit.geonrm = normal;
            hit.tangent = f3(1, 0, 0);
            hit.bitangent = f3(0, 0, 1);
            hit.color = f4(1, 1, 1, 1);
            hit.uv0 = hit.uv1 = f2(0.0f, 0.0f);
            hit.texelDensity = 0.0f;
            statAdd(&stats->shadedHits, 1ull);
            return true;
          }
        }
      }
    }

    if(slot == 0xFFFFFFFFu)
    {
      // ---- environment (gltf_pathtrace.slang:129-156) ----
      if(depth == 0)
      {
        flags &= ~PF_SOLID;  // tryPrimaryMissBackplate: pt.solid = false
        const bool dlss = isDlssFrame(P, F);
        if(isFirstFrame(F, i) || dlss)
          P.firstHit[i] = f4(dir, 0.0f);  // pt.firstHitPos = ray.Direction (pathtrace_functions.h.slang:950)
        if(dlss)
          P.prevHit[i] = f4(dir, 0.0f);  // pt.firstHitPosPrev = ray.Direction (:952-955)
        if(F.fi.flags & B200PT_SCENE_USE_SOLID_BACKGROUND)
        {
          finalizeSample(P, F, i, f3(F.fi.backgroundColor[0], F.fi.backgroundColor[1], F.fi.backgroundColor[2]), false, seed, sampleIdx, qNext, cntNext, stats);
          return false;
        }
      }
      if(flags & PF_SPEC_CAPTURE)
      {
        // a glossy reflection of the first hit went to the sky: fp16 max (gltf_pathtrace.slang:135-143)
        uint2* const sp = &P.dlssSpec[i];
        sp->y = (sp->y & 0xffffu) | ((uint32_t)dlssHalfBits(65504.0f) << 16);
        flags &= ~PF_SPEC_CAPTURE;
      }
      const float4 env = sampleEnvironment(S, F, dir);
      radiance += throughput * computeEnvHitMisWeight(S, F, lastSamplePdf, env.w) * xyz(env);
      finalizeSample(P, F, i, radiance, (flags & PF_SOLID) != 0, seed, sampleIdx, qNext, cntNext, stats);
      return false;
    }

    // ---- hit-attribute fetch ----
    hit = fetchHitState(S, slot, hr.y, hr.z, dir, meta, nodeP);
#ifdef B200PT_DEBUG
    // reference analogue: doDebug at pushConst.mouseCoord (gltf_pathtrace.slang:553-557)
    dbgPixel = ((float)(pixelOf(F, i) % (uint32_t)F.width) == F.pc.mouseCoord[0] && (float)pixelRow(F, pixelOf(F, i)) == F.pc.mouseCoord[1]);
    if(dbgPixel)
      printf("DBG hit t=%.9g rnode=%d prim=%d bary=%.9g %.9g org=%.9g %.9g %.9g dir=%.9g %.9g %.9g seed=%u depth=%d\n", hitT, (int)(meta.x & 0x0fffffffu), (int)meta.y, hr.y, hr.z,
             org.x, org.y, org.z, dir.x, dir.y, dir.z, seed, (int)depth);
#endif
    statAdd(&stats->shadedHits, 1ull);
    return true;
  };
  // ---- section 2: material evaluation (three trilinear texture lookups), emission, unlit ----
  auto shadeMaterial = [&]() -> bool {
    worldFoot = rayConeWorldFootprint(coneWidth, F.pc.pixelAngle, hitT, hit.geonrm, dir);
    int unlit = 0;
    if(onPlane)
    {
      pbrMat = planeMaterial(F);
      if(F.fi.flags & B200PT_SCENE_INFINITE_PLANE_SHADOW_CATCHER)
      {
        // gltf_pathtrace.slang:175-186: the catcher returns before the first-hit captures, the roughness clamp and emission; its light
        // sample is drawn in the next section (the one sampleLights of this kernel), its second half runs after the shadow trace
        catcher = true;
        return true;
      }
    }
    else
    {
      const b200pt_render_node&    node = *nodeP;
      const int                    materialIndex = max(0, node.materialID);
      const float                  texGrad = footprintTexGrad(worldFoot, hit.texelDensity, F.pc.texGradScale);
      const b200pt_shade_material& gmat = S.mats[materialIndex];
      pbrMat = evaluateMaterial<FEAT>(S, gmat, hit, (flags & PF_INSIDE) != 0, texGrad);
      unlit = gmat.unlit;
    }

    if(flags & PF_SPEC_CAPTURE)
    {
      // the first surface behind a glossy reflection of the first hit (:216-223); the shadow catcher returned above, so its plane
      // leaves the capture armed
      uint2* const sp = &P.dlssSpec[i];
      sp->y = (sp->y & 0xffffu) | ((uint32_t)dlssHalfBits(hitT) << 16);
      flags &= ~PF_SPEC_CAPTURE;
    }

    // firefly control: never get sharper than the roughest bounce so far (:267-268)
    misc.x = fmaxf(pbrMat.roughness.x, misc.x);
    misc.y = fmaxf(pbrMat.roughness.y, misc.y);
    pbrMat.roughness = f2(misc.x, misc.y);

    // first-hit capture for the NDC depth output of frame 0 and, on DLSS frames, of every frame (gltf_pathtrace.slang:228-232)
    const bool dlss = isDlssFrame(P, F);
    if(depth == 0 && (isFirstFrame(F, i) || dlss))
      P.firstHit[i] = f4(hit.pos, 1.0f);
    // denoiser guides of the first hit (gltf_pathtrace.slang:240-263): base colour and shading normal / roughness, stored as
    // float16_t by the reference.  (maxRoughness is still 0 at depth 0, so the clamp above left pbrMat.roughness as evaluateMaterial
    // returned it.)
    if(depth == 0 && P.guideA && (F.pc.flags & (B200PT_PT_USE_OPTIX_DENOISER | B200PT_PT_USE_DLSS)))
    {
      auto h16 = [](float x) { return __half2float(__float2half_rn(x)); };
      P.guideA[i] = f4(h16(pbrMat.baseColor.x), h16(pbrMat.baseColor.y), h16(pbrMat.baseColor.z), h16(pbrMat.roughness.x));
      P.guideN[i] = f4(h16(pbrMat.N.x), h16(pbrMat.N.y), h16(pbrMat.N.z), 1.0f);
    }
    if(depth == 0 && dlss)
    {
      // instance motion: the same surface point under the previous frame's objectToWorld (:235-241); the plane does not move
      float3 prev = hit.pos;
      if(!onPlane && F.prevObjectToWorld)
      {
        const uint32_t rnode = meta.x & 0x0fffffffu;
        const float4   objPos = mul_vM(f4(hit.pos, 1.0f), *reinterpret_cast<const Mat4*>(nodeP->worldToObject));
        prev = xyz(mul_vM(f4(xyz(objPos), 1.0f), *reinterpret_cast<const Mat4*>(F.prevObjectToWorld + 16u * rnode)));
      }
      P.prevHit[i] = f4(prev, 1.0f);
      // specular albedo (:246-255): dielectric f0 from the ior pair (pow(x, 2) as the correctly rounded x * x), times the specular
      // colour, clamped to 1.  The hit distance half stays 0: a capture is armed only by a depth-0 BSDF sample, after which depth > 0.
      const float  r = (pbrMat.ior2 - pbrMat.ior1) / (pbrMat.ior2 + pbrMat.ior1);
      const float  f0 = r * r;
      const float3 sc = f3(fminf(f0 * pbrMat.specularColor.x, 1.0f), fminf(f0 * pbrMat.specularColor.y, 1.0f), fminf(f0 * pbrMat.specularColor.z, 1.0f));
      const float3 sa = dlssEnvBRDFApprox2(sc, pbrMat.roughness.x, dot(pbrMat.N, dir));
      P.dlssSpec[i] = make_uint2((uint32_t)dlssHalfBits(sa.x) | ((uint32_t)dlssHalfBits(sa.y) << 16), (uint32_t)dlssHalfBits(sa.z));
    }

    radiance += pbrMat.emissive * throughput;

    if(unlit > 0)
    {
      radiance += pbrMat.baseColor;
      finalizeSample(P, F, i, radiance, (flags & PF_SOLID) != 0, seed, sampleIdx, qNext, cntNext, stats);
      return false;
    }

    return true;
  };
  // the end of sections 3 and 4: the path's next ray and state
  auto storePath = [&]() {
    P.rayO[i] = f4(org, coneWidth);
    P.rayD[i] = f4(normalize(dir), kInfinite);
    P.thr[i] = f4(throughput, lastSamplePdf);
    P.rad[i] = f4(radiance, __uint_as_float(scatterBounces));
    P.misc[i] = f4(misc.x, misc.y, __uint_as_float(flags), __uint_as_float(seed));
  };
  // the path goes on to k_resolve, and its pending shadow ray to the shadow walk
  auto handOff = [&]() {
    queuePush(qPost, cntPost, i);
    if(flags & PF_SHADOW_VALID)
      queuePush(qShadow, cntShadow, i);
  };
  // ---- section 3: in-volume segment, light / environment sample ----
  auto shadeLight = [&]() -> bool {
    flags &= ~(PF_POST_VOLUME | PF_SHADOW_VALID | PF_SHADOW_INSIDE);

    // ---- in-volume segment (pathtrace_functions.h.slang:904-939, 605-672) ----
    if((FEAT & FEAT_VOLUME) && (flags & PF_INSIDE) && !catcher)
    {
      const VolumeMedium vm = unpackMedium(med);
      if(hasVolumeMedium(vm))
      {
        const float3 ext = vm.extinction, sc = vm.scatterCoefficient;
        bool         scattered = false;
        if(maxc(sc) > 0.001f)
        {
          const float maxExt = maxc(ext);
          const float scatterDist = -logf(fmaxf(rnd(seed), 1.0e-10f)) / maxExt;
          if(scatterDist < hitT)
          {
            throughput *= f3(1.0f) - (ext - sc) / maxExt;
            const float3 wi = dir;
            const float3 originBefore = org;
            org = org + dir * scatterDist;
            const float a = rnd(seed), b = rnd(seed);
            dir = sampleHenyeyGreenstein(f2(a, b), vm.scatterAnisotropy, wi);
            lastSamplePdf = henyeyGreensteinPdf(dot(wi, dir), vm.scatterAnisotropy);
            scattered = true;
            scatterBounces++;
            coneWidth += F.pc.pixelAngle * length(org - originBefore);
            // NEE at the scatter point (volumeScatterNEE)
            const DirectLight dl = sampleLights<FEAT>(S, F, org, seed);
            if(dl.pdf > 0.0f)
            {
              const float phasePdf = henyeyGreensteinPdf(dot(wi, dl.direction), vm.scatterAnisotropy);
              const float misWeight = dl.pdf / (dl.pdf + phasePdf);
              // reference: throughput * radianceOverPdf * misWeight * phasePdf * shadowFactor
              P.shC[i] = f4(throughput * dl.radianceOverPdf * misWeight * phasePdf, 0.0f);
              P.shO[i] = f4(org, dl.distance);
              P.shD[i] = f4(dl.direction, 0.0f);
              flags |= PF_SHADOW_VALID | PF_SHADOW_INSIDE;
            }
            flags |= PF_POST_VOLUME;
#ifdef B200PT_DEBUG
            if(dbgPixel)
              printf("DBG scatter n=%d o=%.9g %.9g %.9g d=%.9g %.9g %.9g thr=%.9g %.9g %.9g pdf=%.9g neeC=%.9g %.9g %.9g valid=%d seed=%u\n", (int)scatterBounces, org.x, org.y, org.z, dir.x, dir.y,
                     dir.z, throughput.x, throughput.y, throughput.z, lastSamplePdf, (flags & PF_SHADOW_VALID) ? P.shC[i].x : 0.f, (flags & PF_SHADOW_VALID) ? P.shC[i].y : 0.f,
                     (flags & PF_SHADOW_VALID) ? P.shC[i].z : 0.f, (int)((flags & PF_SHADOW_VALID) != 0), seed);
#endif
          }
          else
            throughput *= expv((f3(maxExt) - ext) * hitT);
        }
        else
          throughput *= expv(ext * -hitT);
        if(scattered)
        {
          storePath();
          handOff();
          return false;
        }
      }
    }

    coneWidth = worldFoot;

    // ---- next-event estimation: one light-or-environment sample, MIS (:316-351) ----
    directLight = sampleLights<FEAT>(S, F, hit.pos, seed);
    if(catcher)
    {
      // handleShadowCatcher, first half (:511-523): the light sample and its shadow ray -- from the plane point itself, unbounded.
      // The shadow factor comes back through the shadow / any-hit kernels in shC; finishPost continues with the second half.
      flags |= PF_CATCHER;
      if(dot(directLight.direction, hit.nrm) > 0.0f && directLight.pdf != 0.0f)
      {
        P.shO[i] = f4(hit.pos, kInfinite);
        P.shD[i] = f4(directLight.direction, 0.0f);
        P.shC[i] = f4(1.0f, 1.0f, 1.0f, 0.0f);
        flags |= PF_SHADOW_VALID;
      }
      P.rayO[i] = f4(hit.pos, coneWidth);  // the incoming direction stays in rayD: the second half looks the environment up along it
      P.misc[i] = f4(misc.x, misc.y, __uint_as_float(flags), __uint_as_float(seed));
      handOff();
      return false;
    }
    nextEventValid = (dot(directLight.direction, hit.nrm) > 0.0f || pbrMat.diffuseTransmissionFactor > 0.0f) && directLight.pdf != 0.0f;
    return true;
  };
  // ---- section 4: BSDF evaluation for the light sample, BSDF sampling, next ray + shadow ray ----
  auto shadeBsdf = [&]() {
    float3 contribution = f3(0.0f);
#ifdef B200PT_DEBUG
    if(dbgPixel)
      printf("DBG shade pos=%.9g %.9g %.9g nrm=%.9g %.9g %.9g gn=%.9g %.9g %.9g N=%.9g %.9g %.9g rough=%.9g %.9g metal=%.9g base=%.9g %.9g %.9g L=%.9g %.9g %.9g lpdf=%.9g valid=%d seed=%u\n",
             hit.pos.x, hit.pos.y, hit.pos.z, hit.nrm.x, hit.nrm.y, hit.nrm.z, hit.geonrm.x, hit.geonrm.y, hit.geonrm.z, pbrMat.N.x, pbrMat.N.y, pbrMat.N.z, pbrMat.roughness.x,
             pbrMat.roughness.y, pbrMat.metallic, pbrMat.baseColor.x, pbrMat.baseColor.y, pbrMat.baseColor.z, directLight.direction.x, directLight.direction.y,
             directLight.direction.z, directLight.pdf, (int)nextEventValid, seed);
#endif
    if(nextEventValid)
    {
      const float    a = rnd(seed), b = rnd(seed), c = rnd(seed);
      const BsdfEval ev = bsdfEvaluate<FEAT>(pbrMat, -dir, directLight.direction, f3(a, b, c));
      if(ev.pdf > 0.0f)
      {
        const float  misWeight = (directLight.pdf == kDirac) ? 1.0f : directLight.pdf / (directLight.pdf + ev.pdf);
        const float3 w = throughput * directLight.radianceOverPdf * misWeight;
        contribution += w * ev.bsdf_diffuse;
        contribution += w * ev.bsdf_glossy;
      }
    }

    // ---- BSDF sampling: next direction + throughput (:357-416) ----
    {
      const float      a = rnd(seed), b = rnd(seed), c = rnd(seed);
      const BsdfSample sd = bsdfSample<FEAT>(pbrMat, -dir, f3(a, b, c));
#ifdef B200PT_DEBUG
      if(dbgPixel)
        printf("DBG sample xi=%.9g %.9g %.9g k2=%.9g %.9g %.9g bop=%.9g %.9g %.9g pdf=%.9g ev=%d contrib=%.9g %.9g %.9g\n", a, b, c, sd.k2.x, sd.k2.y, sd.k2.z, sd.bsdf_over_pdf.x,
               sd.bsdf_over_pdf.y, sd.bsdf_over_pdf.z, sd.pdf, sd.event_type, contribution.x, contribution.y, contribution.z);
#endif
      throughput *= sd.bsdf_over_pdf;
      dir = sd.k2;
      lastSamplePdf = sd.pdf;
      // DLSS: a glossy or mirror reflection of the first hit arms the specular hit-distance capture (:370-377)
      if(depth == 0 && (sd.event_type == BSDF_EVENT_GLOSSY_REFLECTION || sd.event_type == (BSDF_EVENT_IMPULSE | BSDF_EVENT_REFLECTION)) && isDlssFrame(P, F))
        flags |= PF_SPEC_CAPTURE;
      if(sd.event_type != BSDF_EVENT_ABSORB)
      {
        const float3 offsetDir = dot(dir, hit.geonrm) > 0 ? hit.geonrm : -hit.geonrm;
        org = safeOffsetRay(hit.pos, offsetDir);
        if((FEAT & (FEAT_TRANSMISSION | FEAT_DIFFUSE_TRANSMISSION)) && (sd.event_type & BSDF_EVENT_TRANSMISSION))
        {
          flags ^= PF_INSIDE;
          if((FEAT & FEAT_VOLUME) && (flags & PF_INSIDE))
            med = packMedium(makeVolumeMedium(pbrMat), med.w >> 16);
        }
      }
      else
        depth = (uint32_t)F.pc.maxDepth;
    }

    // ---- shadow ray for the delayed NEE visibility test (:418-426) ----
    if(nextEventValid)
    {
      const bool   forward = dot(directLight.direction, hit.nrm) > 0.0f;
      const float3 sDir = forward ? hit.geonrm : -hit.geonrm;
      const float3 sBase = forward ? hit.shadowPos : hit.pos;
      P.shO[i] = f4(safeOffsetRay(sBase, sDir), directLight.distance);
      P.shD[i] = f4(directLight.direction, 0.0f);
      P.shC[i] = f4(contribution, 0.0f);
      flags |= PF_SHADOW_VALID;
    }

    flags = (flags & ~PF_DEPTH_MASK) | (depth & PF_DEPTH_MASK);
    storePath();
    P.medium[i] = med;
    handOff();
  };
  for(uint32_t base = blockIdx.x * blockDim.x; base < count; base += stride)
  {
    bool alive = base + threadIdx.x < count;
    __syncthreads();
    if(alive)
      alive = shadeLoad(base + threadIdx.x);
    if(alive)
      alive = shadeMaterial();
    if(alive)
      alive = shadeLight();
    if(alive)
      shadeBsdf();
  }
}

// pathTrace() tail for every path that survived shading: delayed NEE visibility (TraceShadow), Russian
// roulette, depth++ (gltf_pathtrace.slang:462-485).  Same persistent-warp scheme as k_trace; paths without a
// shadow ray finish immediately and their lanes are refilled.
__device__ void finishPost(const PathState& P, const DevScene& S, const FrameParams& F, uint32_t i, uint32_t flags, uint32_t seed, bool haveShadow, float3 Tfac,
                           uint32_t* qNext, uint32_t* cntNext, DevStats* stats)
{
  const float4 misc = P.misc[i];
  const float4 rad4 = P.rad[i];
  float3       radiance = xyz(rad4);
  const float4 thr4 = P.thr[i];
  float3       throughput = xyz(thr4);
  auto         endSample = [&]() { finalizeSample(P, F, i, radiance, (flags & PF_SOLID) != 0, seed, P.medium[i].w >> 16, qNext, cntNext, stats); };
  if(flags & PF_CATCHER)
  {
    // handleShadowCatcher, second half (pathtrace_functions.h.slang:525-553): lit plane points show the environment behind them and
    // end the path; shadowed ones show it darkened and continue with bsdfSampleSimple -- eEarlyContinue: no roulette, no depth++
    const float3 shadowFactor = haveShadow ? xyz(P.shC[i]) * Tfac : f3(1.0f);
    const float4 ro = P.rayO[i];
    const float3 hitPos = xyz(ro), dir = xyz(P.rayD[i]);
    const float4 env = sampleEnvironment(S, F, dir);
    const float3 envColor = xyz(env);
    flags &= ~(PF_CATCHER | PF_POST_VOLUME | PF_SHADOW_VALID | PF_SHADOW_INSIDE);
    if(shadowFactor.x == 1.0f && shadowFactor.y == 1.0f && shadowFactor.z == 1.0f)
    {
      radiance += throughput * computeEnvHitMisWeight(S, F, thr4.w, env.w) * envColor;
      endSample();
      return;
    }
    radiance += envColor * shadowFactor;
    radiance -= envColor * (f3(1.0f) - shadowFactor) * F.fi.shadowCatcherDarkenAmount;
    const PbrMaterial pm = planeMaterial(F);
    const float       a = rnd(seed), b = rnd(seed), c = rnd(seed);
    const BsdfSample  sd = bsdfSampleSimple(pm, -dir, f3(a, b, c));
    if(sd.event_type == BSDF_EVENT_ABSORB)
    {
      endSample();
      return;
    }
    const float3 offsetDir = dot(sd.k2, pm.N) > 0 ? pm.N : -pm.N;
    throughput *= sd.bsdf_over_pdf;
    P.rayO[i] = f4(safeOffsetRay(hitPos, offsetDir), ro.w);
    P.rayD[i] = f4(normalize(sd.k2), kInfinite);
    P.thr[i] = f4(throughput, sd.pdf);
    P.rad[i] = f4(radiance, rad4.w);
    P.misc[i] = f4(misc.x, misc.y, __uint_as_float(flags), __uint_as_float(seed));
    queuePush(qNext, cntNext, i);
    return;
  }
  if(haveShadow)
    radiance += xyz(P.shC[i]) * Tfac;
  uint32_t depth = flags & PF_DEPTH_MASK;
  // Russian roulette: inside a volume only after VOLUME_FREE_BUDGET scatters (pathtrace_functions.h.slang:925-931), on a surface
  // from depth 3 (gltf_pathtrace.slang:476-485)
  const bool volume = (flags & PF_POST_VOLUME) != 0;
  const bool roulette = volume ? __float_as_uint(rad4.w) >= 64u : depth >= 3u;
  bool       alive = true;
  if(roulette)
  {
    const float rrPcont = fminf(maxc(throughput) + 0.001f, 0.95f);
    if(rnd(seed) >= rrPcont)
      alive = false;
    else
      throughput /= rrPcont;
  }
  if(alive && !volume)
  {
    depth++;
    if((int)depth >= F.pc.maxDepth)
      alive = false;
  }
  if(!alive)
  {
    endSample();
    return;
  }
  flags = (flags & ~(PF_DEPTH_MASK | PF_POST_VOLUME | PF_SHADOW_VALID | PF_SHADOW_INSIDE)) | (depth & PF_DEPTH_MASK);
  if(haveShadow)
    P.rad[i] = f4(radiance, rad4.w);
  if(roulette)
    P.thr[i] = f4(throughput, thr4.w);
  P.misc[i] = f4(misc.x, misc.y, __uint_as_float(flags), __uint_as_float(seed));
  queuePush(qNext, cntNext, i);
}

// IRaytracer::TraceShadow, geometry part, for every path with a pending NEE shadow ray: ONE walk of the scene tree along
// the whole segment; any FORCE_OPAQUE occluder ends the query (raytracer_interface.h.slang:181-184), otherwise the kCand
// nearest non-opaque candidates are written out for k_alpha<true>.  Same persistent-warp scheme as k_trace.
// candInfo.x of a shadow ray that an opaque occluder ended (raytracer_interface.h.slang:181-184)
constexpr uint32_t kShadowOccluded = 0x80000000u;
template <bool OMM, bool CAPS>
__global__ void __launch_bounds__(kWalkBlock, kWalkCtasPerSM) k_shadow(PathState P, DevScene S, const uint32_t* __restrict__ q, const uint32_t* __restrict__ cntIn,
                                                                       uint32_t* workCounter, uint32_t* qAlpha, uint32_t* cntAlpha, DevStats* stats, int mode)
{
  const bool cont = (mode & TRACE_CONT) != 0;
  int        phase = 0;  // 0: occlusion query against the opaque-only tree, 1: candidates from the non-opaque tree
  auto       start = [&](TravState& T, int path) {
    const float4 so = P.shO[path];
    const float4 sd = P.shD[path];
    if(!cont)
    {
      phase = 0;
      T.init(S.bvhO, xyz(so), xyz(sd), 0.0f, so.w, false, true, false, 0.f, 0u, false);
    }
    else
    {
      phase = 1;
      T.init(S.bvhA, xyz(so), xyz(sd), 0.0f, so.w, false, true, true, P.cand[kCand - 1][path].x, P.candInfo[path].y, true);
    }
  };
  auto finish = [&](TravState& T, const Cand* cand, int path) {
    if(phase == 0 && T.best.slot == 0xFFFFFFFFu && S.hasAlpha)
    {
      // no opaque occluder: the non-opaque candidates of the segment, nearest first
      // With opacity micromaps an OPAQUE micro-triangle anywhere on the segment ends the query like a FORCE_OPAQUE occluder
      // (a committed hit, raytracer_interface.h.slang:181-184), so the walk must not stop looking behind the 4th candidate.
      phase = 1;
      T.init(S.bvhA, T.org, T.dir, 0.0f, T.tmax, false, true, false, 0.f, 0u, !OMM);
      return false;
    }
    uint2 info = make_uint2(0u, 0u);
    if(T.best.slot != 0xFFFFFFFFu)
      info.x = kShadowOccluded;
    else
    {
      const int n = T.collectN;
      info = make_uint2((uint32_t)n, n > 0 ? cand[(n - 1) * kWalkBlock].gid : 0u);
      // every candidate a cap (opacity 1, transmission <= 0.01: it blocks the ray) or a hole (opacity 0: never passes): k_alpha<true>'s
      // loop here, without texels, in a ray's first round (a continuation round folds the transmission parked by the previous one)
      if(CAPS && !cont && n > 0 && knownOpacities(cand, n))
      {
        uint32_t* const seedOut = reinterpret_cast<uint32_t*>(&P.misc[path]) + 3;
        uint32_t        seed = *seedOut;
        bool            blocked = false;
#pragma unroll
        for(int i = 0; i < kCand; i++)
          if(i < n && !blocked && rnd(seed) < ((cand[i * kWalkBlock].slot & kCandCap) ? 1.0f : 0.0f))
            blocked = true;
        if(blocked || n < kCand)
        {
          const float4 c = P.shC[path];
          P.shC[path] = f4(xyz(c) * (blocked ? f3(0.0f) : f3(1.0f)), c.w);
          *seedOut = seed;
          P.candInfo[path] = info;
          return true;
        }
      }
      writeCandidates<CAPS>(P, path, cand, n);
    }
    P.candInfo[path] = info;
    // (a continuation path always goes back to k_alpha: its running transmission is parked and must be folded)
    if((info.x != 0u && info.x != kShadowOccluded) || cont)
      queuePush(qAlpha, cntAlpha, (uint32_t)path);
    return true;
  };
  // (only the non-opaque triangles of phase 1 consult the micromaps and the caps)
  walkQueue<OMM, CAPS, 2>(q, *cntIn, workCounter, S.bvhA, stats, cont, start, finish);
}

// ---- material-sorted shade queue (north star: "material-sorted shade queues to tame divergence") -------------------------
// Counting sort of the bounce's path queue by the material of the hit (misses last): k_sort_count builds the histogram,
// k_sort_scan turns it into bucket cursors, k_sort_scatter writes the queue bucket by bucket.  Histogram and offsets are
// aggregated per block in shared memory (a handful of buckets, millions of paths: one global atomic per path would serialise
// on the bucket counters).  Paths are independent, so the order inside a bucket (not deterministic) does not change any pixel.
constexpr int kSortMaxBuckets = 1024;
constexpr int kSortItems = 4;  // paths per thread per pass

// the bucket of a path: the material of its hit, misses last
__device__ __forceinline__ uint32_t shadeKey(const PathState& P, const DevScene& S, uint32_t path, uint32_t nb)
{
  const uint32_t slot = __float_as_uint(P.hit[path].w);
  return slot == 0xFFFFFFFFu ? nb - 1u : min(__ldg(&S.matOfSlot[slot]), nb - 2u);
}

__global__ void __launch_bounds__(256) k_sort_count(PathState P, DevScene S, const uint32_t* __restrict__ q, const uint32_t* __restrict__ cntIn, uint32_t* bucketCount, uint32_t nb)
{
  __shared__ uint32_t sCnt[kSortMaxBuckets];
  for(uint32_t b = threadIdx.x; b < nb; b += blockDim.x)
    sCnt[b] = 0;
  __syncthreads();
  const uint32_t count = *cntIn;
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < count; k += stride)
    atomicAdd(&sCnt[shadeKey(P, S, q[k], nb)], 1u);
  __syncthreads();
  for(uint32_t b = threadIdx.x; b < nb; b += blockDim.x)
    if(sCnt[b])
      atomicAdd(&bucketCount[b], sCnt[b]);
}

// exclusive scan of the (few) bucket counts into cursors; the counts are zeroed for the next bounce
__global__ void __launch_bounds__(1024) k_sort_scan(uint32_t* bucketCount, uint32_t* bucketCursor, uint32_t nb)
{
  __shared__ uint32_t s[kSortMaxBuckets];
  const uint32_t      t = threadIdx.x;
  s[t] = t < nb ? bucketCount[t] : 0u;
  __syncthreads();
  for(uint32_t d = 1; d < kSortMaxBuckets; d <<= 1)
  {
    const uint32_t v = t >= d ? s[t - d] : 0u;
    __syncthreads();
    s[t] += v;
    __syncthreads();
  }
  if(t < nb)
  {
    bucketCursor[t] = s[t] - bucketCount[t];
    bucketCount[t] = 0u;
  }
}

__global__ void __launch_bounds__(256) k_sort_scatter(PathState P, DevScene S, const uint32_t* __restrict__ q, const uint32_t* __restrict__ cntIn, uint32_t* bucketCursor,
                                                      uint32_t* __restrict__ qSorted, uint32_t nb)
{
  __shared__ uint32_t sCnt[kSortMaxBuckets], sBase[kSortMaxBuckets];
  const uint32_t      count = *cntIn;
  const uint32_t      chunk = blockDim.x * kSortItems;
  for(uint32_t base = blockIdx.x * chunk; base < count; base += gridDim.x * chunk)  // block-uniform trip count
  {
    for(uint32_t b = threadIdx.x; b < nb; b += blockDim.x)
      sCnt[b] = 0;
    __syncthreads();
    uint32_t path[kSortItems], key[kSortItems], off[kSortItems];
#pragma unroll
    for(int i = 0; i < kSortItems; i++)
    {
      const uint32_t k = base + (uint32_t)i * blockDim.x + threadIdx.x;
      key[i] = 0xFFFFFFFFu;
      if(k < count)
      {
        path[i] = q[k];
        key[i] = shadeKey(P, S, path[i], nb);
        off[i] = atomicAdd(&sCnt[key[i]], 1u);
      }
    }
    __syncthreads();
    for(uint32_t b = threadIdx.x; b < nb; b += blockDim.x)
      if(sCnt[b])
        sBase[b] = atomicAdd(&bucketCursor[b], sCnt[b]);
    __syncthreads();
#pragma unroll
    for(int i = 0; i < kSortItems; i++)
      if(key[i] != 0xFFFFFFFFu)
        qSorted[sBase[key[i]] + off[i]] = path[i];
    __syncthreads();
  }
}

// pathTrace() tail for every path that survived shading (gltf_pathtrace.slang:462-485), one thread per path: the
// delayed NEE contribution (already scaled by the any-hit transmission in k_alpha<true>; an opaque occluder
// zeroes it here), Russian roulette and depth++ in finishPost.
__global__ void __launch_bounds__(256) k_resolve(PathState P, DevScene S, const __grid_constant__ FrameParams F, const uint32_t* __restrict__ q, const uint32_t* __restrict__ cntIn,
                                                 uint32_t* qNext, uint32_t* cntNext, DevStats* stats)
{
  const uint32_t count = *cntIn;
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < count; k += stride)
  {
    const uint32_t path = q[k];
    const float4   misc = P.misc[path];
    const uint32_t flags = __float_as_uint(misc.z);
    const uint32_t seed = __float_as_uint(misc.w);
    const bool     haveShadow = (flags & PF_SHADOW_VALID) != 0;
    float3         vis = f3(1.0f);
    if(haveShadow && (P.candInfo[path].x & kShadowOccluded))
      vis = f3(0.0f);
#ifdef B200PT_DEBUG
    if(haveShadow && (float)(pixelOf(F, path) % (uint32_t)F.width) == F.pc.mouseCoord[0] && (float)pixelRow(F, pixelOf(F, path)) == F.pc.mouseCoord[1])
      printf("DBG shadow occluded=%d\n", (int)(vis.x == 0.0f));
#endif
    finishPost(P, S, F, path, flags, seed, haveShadow, vis, qNext, cntNext, stats);
  }
}

// processPixel tail: mean over the frame's samples + running mean over frames (gltf_pathtrace.slang:596,619-630); on the
// first frame also the NDC depth of the last sample's first hit (:600-616; Vulkan [0,1] range, 1 = far / miss).  A DLSS frame
// replaces the image like a first frame (:619-622).  With views, slot block v updates view v's image: view 0 is `accum` / `ndcDepth`,
// view v > 0 starts at viewAccum / viewDepth + (v - 1) * pixels.
__global__ void __launch_bounds__(256) k_accumulate(PathState P, const __grid_constant__ FrameParams F, float4* __restrict__ accum, float* __restrict__ ndcDepth,
                                                    float4* __restrict__ viewAccum, float* __restrict__ viewDepth)
{
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < F.pixels * (uint32_t)F.views; i += stride)
  {
    float4* const out = i < F.pixels ? accum + i : viewAccum + (i - F.pixels);
    float4        img = f4(0.f, 0.f, 0.f, 0.f);
    // the frames of a batch are folded in frame order, each with the sample counts its own push constants would have carried
    for(int b = 0; b < F.batch; b++)
    {
      const float4 c = P.pixSum[i + (uint32_t)b * F.pixels] / (float)F.pc.numSamples;
      if(b == 0 && (F.pc.flags & (B200PT_PT_FIRST_FRAME | B200PT_PT_USE_DLSS)))
      {
        img = c;
        if(ndcDepth && (F.pc.flags & B200PT_PT_FIRST_FRAME))
        {
          const float4 fh = P.firstHit[i];
          float        d = 1.0f;
          if(fh.w > 0.0f)
          {
            const Mat4&  vp = *reinterpret_cast<const Mat4*>(cameraOf(F, i).viewProjMatrix);
            const float4 clip = mul_vM(f4(fh.x, fh.y, fh.z, 1.0f), vp);
            d = clip.z / clip.w;
          }
          *(i < F.pixels ? ndcDepth + i : viewDepth + (i - F.pixels)) = d;
        }
      }
      else
      {
        if(b == 0)
          img = *out;
        const int    totalSamples = F.pc.totalSamples + b * F.pc.numSamples;
        const float  total = (float)totalSamples, n = (float)F.pc.numSamples;
        const float  after = (float)(totalSamples + F.pc.numSamples);
        const float4 old = img;
        img = f4((old.x * total + c.x * n) / after, (old.y * total + c.y * n) / after, (old.z * total + c.z * n) / after, (old.w * total + c.w * n) / after);
      }
    }
    *out = img;
  }
}

// OutputImage::eOptixAlbedoNormal (gltf_pathtrace.slang:653-670): per pixel the LAST sample's guide albedo and its shading normal in
// camera space, compressed to 32 bits.  compressUnitVec is nvshaders code (external): restated as the octahedral 2 x 16-bit encoding it
// implements (Engelhardt & Dachsbacher 2008): project onto |x| + |y| + |z| = 1, fold the lower hemisphere, 16 bits per axis.
PT_HD uint32_t compressUnitVec(float3 nv)
{
  if(!(fabsf(nv.x) < 3.0e38f))  // NaN / infinity
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

__global__ void __launch_bounds__(256) k_guide(PathState P, const __grid_constant__ FrameParams F, float4* __restrict__ guide)
{
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < F.pixels; i += stride)
  {
    const uint32_t slot = i + (uint32_t)(F.batch - 1) * F.pixels;  // the newest frame of the batch
    const float4   a = P.guideA[slot], n = P.guideN[slot];
    float3         camN = f3(0.0f, 0.0f, 1.0f);  // primary miss: a valid forward-facing normal (:658-660)
    if(n.w > 0.0f)
    {
      // mul(float3x3(viewMatrix), worldNormal) on the glm bytes (SURVEY.md section 8, convention note): M_glm^T * n
      const float* m = cameraOf(F, slot).viewMatrix;
      camN = normalize(f3((m[0] * n.x + m[1] * n.y) + m[2] * n.z, (m[4] * n.x + m[5] * n.y) + m[6] * n.z, (m[8] * n.x + m[9] * n.y) + m[10] * n.z));
    }
    guide[i] = f4(a.x, a.y, a.z, __uint_as_float(compressUnitVec(camN)));
  }
}

// The six DLSS guide images of processPixel (gltf_pathtrace.slang:628-651) for the newest frame, each plane in its format
// (src/dlss.cpp:61-66): albedo RGBA8, specular albedo RGBA16F, normal / roughness RGBA16F, motion RG16F, depth R16F, specular hit
// distance R16F.
struct DlssPlanes
{
  uint32_t* albedo;
  uint2*    specAlbedo;
  uint2*    normalRough;
  uint32_t* motion;
  uint16_t* depth;
  uint16_t* specHitDist;
};

__global__ void __launch_bounds__(256) k_dlss_guides(PathState P, const __grid_constant__ FrameParams F, DlssPlanes out)
{
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < F.pixels; i += stride)
  {
    const uint32_t slot = i + (uint32_t)(F.batch - 1) * F.pixels;
    const float4   a = P.guideA[slot], n = P.guideN[slot];
    const bool     solid = P.pixSum[slot].w > 0.0f;  // sampleResult.radiance.w > 0 (the firefly clamp scales it by a positive factor)
    const Camera         cam = cameraOf(F, slot);
    const DlssGuidePixel g = dlssPackGuides(xyz(a), f4(n.x, n.y, n.z, a.w), P.dlssSpec[slot], xyz(P.firstHit[slot]), xyz(P.prevHit[slot]), solid,
                                            cam.viewProjMatrix, cam.prevMVP, f2(F.fi.imageSize[0], F.fi.imageSize[1]));
    out.albedo[i] = g.albedo;
    out.specAlbedo[i] = make_uint2((uint32_t)g.specAlbedo[0] | ((uint32_t)g.specAlbedo[1] << 16), (uint32_t)g.specAlbedo[2] | ((uint32_t)g.specAlbedo[3] << 16));
    out.normalRough[i] = make_uint2((uint32_t)g.normalRough[0] | ((uint32_t)g.normalRough[1] << 16), (uint32_t)g.normalRough[2] | ((uint32_t)g.normalRough[3] << 16));
    out.motion[i] = (uint32_t)g.motion[0] | ((uint32_t)g.motion[1] << 16);
    out.depth[i] = g.depth;
    out.specHitDist[i] = g.specHitDist;
  }
}

// snapshot_prev_transforms.comp.slang: the render nodes' objectToWorld before a transform update overwrites them
// (world_matrix_io.h.slang:65-75), one thread per render node
__global__ void __launch_bounds__(256) k_snapshot_prev_transforms(const b200pt_render_node* __restrict__ nodes, float* __restrict__ prev, uint32_t n)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i >= n)
    return;
  // render nodes are 136 bytes apart, so their matrices are only 8-byte aligned: no 16-byte loads
  const float* src = nodes[i].objectToWorld;
  float*       dst = prev + 16u * i;
  for(int k = 0; k < 16; k++)
    dst[k] = src[k];
}

// traceSelectionRay (pathtrace_functions.h.slang:813-820) for every pixel of the first frame: the pixel-centre ray
// (no jitter, no depth of field), IRaytracer::TraceLow semantics (raytracer_interface.h.slang:124-137: every triangle
// opaque, no culling), object id = render node + 1, 0 on a miss.  One walk per thread; runs once per accumulation.  With views, slot
// block v writes view v's ids: view 0 to `objectId`, view v > 0 from viewIds + (v - 1) * pixels.
__global__ void __launch_bounds__(128) k_select(DevScene S, const __grid_constant__ FrameParams F, uint32_t* __restrict__ objectId, uint32_t* __restrict__ viewIds,
                                                DevStats* stats)
{
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < F.pixels * (uint32_t)F.views; i += stride)
  {
    const uint32_t px = i % F.pixels;
    float3         org, dir;
    getRay(F, cameraOf(F, i), px % (uint32_t)F.width, pixelRow(F, px), f2(0.5f, 0.5f), org, dir);
    TravState T;
    uint2     stack[TravState::kStackSize];
    Cand      cand[1];
    T.init(S.bvh, org, dir, 0.0f, kInfinite, false, false, false, 0.f, 0u);
    while(!T.step<1, true>(stack, kPostponeShift, cand, 1))
    {
    }
    if(T.overflow)
      atomicOr(&stats->errorFlags, 1ull);
    *(i < F.pixels ? objectId + i : viewIds + (i - F.pixels)) = (T.best.slot != 0xFFFFFFFFu) ? (S.triMeta[T.best.slot].x & 0x0fffffffu) + 1u : 0u;
  }
}

// ---- BVH construction on the device (lbvh.cuh) --------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_lbvh_bounds(LbvhWork W)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i < W.m)
    lbvhBounds(i, W);
}
__global__ void __launch_bounds__(256) k_lbvh_morton(LbvhWork W)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i < W.M)
    lbvhMorton(i, W);
}
__global__ void __launch_bounds__(256) k_lbvh_bitonic(unsigned long long* keys, uint32_t n, uint32_t j, uint32_t k)
{
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if(t < n)
    bitonicStep(t, keys, j, k);
}
__global__ void __launch_bounds__(256) k_lbvh_hierarchy(LbvhWork W)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i + 1 < W.m)
    lbvhHierarchy(i, W);
}
__global__ void __launch_bounds__(256) k_lbvh_fit(LbvhWork W)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i < W.m)
    lbvhFit(i, W);
}
__global__ void __launch_bounds__(128) k_lbvh_emit(LbvhWork W, const int2* queueIn, uint32_t count, int2* queueOut)
{
  const uint32_t q = blockIdx.x * blockDim.x + threadIdx.x;
  if(q < count)
    lbvhEmit(q, W, queueIn, queueOut);
}

// ---- BVH refit after a transform update (refit.cuh) ------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_refit_tris(float* tris, uint2* triMeta, uint32_t n, const b200pt_render_node* nodes, const DevPrim* prims)
{
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
    refitTriangle(i, tris, triMeta, nodes, prims);
}

__global__ void __launch_bounds__(128) k_refit_level(float* nodes, const float* tris, float4* nodeBox, uint32_t first, uint32_t count)
{
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < count; i += stride)
    refitNode(first + i, nodes, tris, nodeBox);
}

// ---- tone mapping + 8-bit encode (tonemap.cuh): HBM-bound, 16 B read + 4 B written per pixel (+ 16 B read for the histogram) ----
__global__ void __launch_bounds__(256) k_tm_histogram(const float4* __restrict__ img, uint32_t n, uint32_t* __restrict__ hist)
{
  __shared__ uint32_t s_h[kTmBins];
  for(int i = threadIdx.x; i < kTmBins; i += blockDim.x)
    s_h[i] = 0u;
  __syncthreads();
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
  {
    const float4 c = __ldg(&img[i]);
    atomicAdd(&s_h[tmBin(0.2126f * c.x + 0.7152f * c.y + 0.0722f * c.z)], 1u);
  }
  __syncthreads();
  for(int i = threadIdx.x; i < kTmBins; i += blockDim.x)
    if(s_h[i])
      atomicAdd(&hist[i], s_h[i]);
}

// log-average luminance over the bins above black -> exposure factor (integer counts, fixed summation order: deterministic)
__global__ void k_tm_exposure(const uint32_t* __restrict__ hist, float baseExposure, float* __restrict__ out)
{
  if(blockIdx.x == 0 && threadIdx.x == 0)
  {
    double sum = 0.0, cnt = 0.0;
    for(int b = 1; b < kTmBins; b++)
    {
      const double centre = (double)kTmMinLog + ((double)b + 0.5) * (double)(kTmMaxLog - kTmMinLog) / (double)kTmBins;
      sum += centre * (double)hist[b];
      cnt += (double)hist[b];
    }
    *out = cnt > 0.0 ? baseExposure * (float)(0.18 / exp2(sum / cnt)) : baseExposure;
  }
}

__global__ void __launch_bounds__(256) k_tonemap(const float4* __restrict__ img, uchar4* __restrict__ out, int width, int rows, int y0, int fullHeight,
                                                 const __grid_constant__ b200pt_tonemapper tm, const float* __restrict__ exposure)
{
  const uint32_t n = (uint32_t)width * (uint32_t)rows, stride = gridDim.x * blockDim.x;
  const float    ex = *exposure;
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
  {
    const float4 c = __ldg(&img[i]);
    const int    x = (int)(i % (uint32_t)width), y = y0 + (int)(i / (uint32_t)width);
    const float3 r = tonemapPixel(tm, ex, f3(c.x, c.y, c.z), ((float)x + 0.5f) / (float)width, ((float)y + 0.5f) / (float)fullHeight);
    out[i] = make_uchar4((unsigned char)tmUnorm8(r.x), (unsigned char)tmUnorm8(r.y), (unsigned char)tmUnorm8(r.z), (unsigned char)tmUnorm8(c.w));
  }
}

// ---- animation feed (animate.cuh): morph.comp.slang / skinning.comp.slang, one thread per vertex like the reference's
// ANIMATION_WORKGROUP_SIZE = 256 dispatches; HBM-bound (<= 72 B read + 40 B written per vertex, matrices stay in L1) -------------
__global__ void __launch_bounds__(256) k_morph(MorphTaskDev T)
{
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if(v < T.vertexCount)
    morphVertex(T, v);
}

__global__ void __launch_bounds__(256) k_skin(SkinTaskDev T)
{
  const uint32_t v = blockIdx.x * blockDim.x + threadIdx.x;
  if(v < T.vertexCount)
    skinVertex(T, v);
}

__global__ void __launch_bounds__(256) k_propagate_level(const float* __restrict__ local, float* world, const int* __restrict__ parents, const int* __restrict__ topo,
                                                         uint32_t levelOffset, uint32_t levelCount)
{
  const uint32_t ti = blockIdx.x * blockDim.x + threadIdx.x;
  if(ti < levelCount)
    propagateNode(local, world, parents, topo, levelOffset, ti);
}

__global__ void __launch_bounds__(256) k_update_render_nodes(const float* __restrict__ world, const RenderNodeMapping* __restrict__ mappings,
                                                             const float* __restrict__ instLocal, b200pt_render_node* out, uint32_t n)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i < n)
    updateRenderNode(world, mappings, instLocal, out, i);
}

__global__ void __launch_bounds__(256) k_regather_shade(ShadeRec* recs, DevPrim P, uint32_t triCount)
{
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if(t < triCount)
    regatherShadeRec(recs + t, P, t);
}

// ---- in-place scene edits (b200pt_update_materials / b200pt_update_node_materials): the tables changed, no triangle changed
// TRI_OPAQUE, so the trees' shapes stay and only what the materials decide is rewritten -------------------------------------
// the flag nibble of every triangle record (and its triMeta copy) from its node's material, TRI_FLIPPED kept; with matOfSlot,
// also the slot's material index
__global__ void __launch_bounds__(256) k_retag_tris(float* tris, uint2* triMeta, uint32_t* matOfSlot, uint32_t n, const b200pt_render_node* nodes,
                                                    const b200pt_shade_material* mats)
{
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
  {
    float*         T = tris + (size_t)i * 12;
    const uint32_t w0 = __float_as_uint(T[3]), rnode = w0 & 0x0fffffffu;
    const uint32_t mat = materialOf(nodes[rnode]);
    const uint32_t w = rnode | ((triFlags(mats[mat]) | ((w0 >> 28) & TRI_FLIPPED)) << 28);
    T[3] = __uint_as_float(w);
    triMeta[i].x = w;
    if(matOfSlot)
      matOfSlot[i] = mat;
  }
}

// the alpha-test records of the non-opaque triangles (slots base .. base + n - 1 of the shadow rays' triangle array)
__global__ void __launch_bounds__(256) k_gather_alpha(AlphaRec* recs, const uint2* __restrict__ metaS, uint32_t base, uint32_t n, DevScene S)
{
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += stride)
  {
    const uint2                meta = metaS[base + k];
    const b200pt_render_node&  node = S.nodes[meta.x & 0x0fffffffu];
    const DevPrim              P = S.prims[node.renderPrimID];
    const DevTex*              tex = S.textures;
    auto                       level0 = [tex](int t) { return tex[t].texels + tex[t].levelOfs[0]; };
    recs[k] = alphaRecOf(S.mats[materialOf(node)], S.texInfos, tex, (uint32_t)S.numTextures, level0, P.uv0, P.uv1, P.col, P.idx[meta.y * 3],
                         P.idx[meta.y * 3 + 1], P.idx[meta.y * 3 + 2]);
  }
}

// the alpha caps and holes of the alpha records (alpha_caps.cuh), one thread per (record, grid cell of kCapLevel): the cap
// micro-triangles of record r are OR-ed into bits[r * 2 * kCapWords ...], its holes into the kCapWords words behind them (zeroed by the
// caller); shadowOk[r]: the record's material may cap a shadow ray
#pragma nv_exec_check_disable
__global__ void __launch_bounds__(256) k_cap_bake(const AlphaRec* __restrict__ recs, uint32_t n, uint32_t* bits, uint8_t* shadowOk)
{
  constexpr uint32_t cells = 2u * kCapMicro;
  const uint64_t     total = (uint64_t)n * cells, stride = (uint64_t)gridDim.x * blockDim.x;
  for(uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride)
  {
    const uint32_t rec = (uint32_t)(i / cells), k = (uint32_t)(i % cells);
    const AlphaRec r = loadAlphaRec(recs + rec);
    if(k == 0)
      shadowOk[rec] = r.transmission <= 0.01f ? 1 : 0;
    const int tpr = (r.w0 + 3) >> 2;
    auto      alpha8 = [&](int x, int y) { return (int)__ldg(r.lv0 + (((y >> 2) * tpr + (x >> 2)) << 4) + ((y & 3) << 2) + (x & 3)).w; };
    auto      wrap = [](int i, int m, int mode) { return wrapFast(i, m, mode); };
    uint32_t  idx;
    bool      cap, hole;
    if(capBakeCell(k, r.uv, r.w0, r.h0, r.wrap, r.factor, r.cutoff, r.modeFlags, r.colA, r.lv0 != nullptr, alpha8, wrap, idx, cap, hole) && (cap || hole))
      atomicOr(&bits[(size_t)rec * 2 * kCapWords + (hole ? kCapWords : 0u) + (idx >> 5)], 1u << (idx & 31u));
  }
}

// ---- ray-level API (parity tests / traversal micro-benchmark): the rays run through the PRODUCTION kernels
// (k_trace / k_shadow -> k_alpha -> continuation round -> k_alpha) on a scratch path pool -------------------------
// rays: recordFloat4s float4 per record, the first two the ray
__global__ void __launch_bounds__(256) k_rays_load(PathState P, const float4* __restrict__ rays, uint32_t recordFloat4s, uint32_t n, const uint32_t* __restrict__ seeds,
                                                   uint32_t* q, uint32_t* cnt, int shadow)
{
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
  {
    const float4 o = rays[i * recordFloat4s], d = rays[i * recordFloat4s + 1];
    if(!shadow)
    {
      P.rayO[i] = o;  // .w = tmin (TRACE_TMIN)
      P.rayD[i] = d;  // .w = tmax
    }
    else
    {
      P.shO[i] = f4(o.x, o.y, o.z, d.w);
      P.shD[i] = f4(d.x, d.y, d.z, 0.0f);
      P.shC[i] = f4(1.0f, 1.0f, 1.0f, 0.0f);
    }
    P.misc[i] = f4(0.0f, 0.0f, __uint_as_float(shadow ? PF_SHADOW_VALID : 0u), __uint_as_float(seeds ? seeds[i] : 0u));
    P.candInfo[i] = make_uint2(0u, 0u);
    q[i] = i;
  }
  if(blockIdx.x == 0 && threadIdx.x == 0)
    *cnt = n;
}

__global__ void __launch_bounds__(256) k_rays_store(PathState P, DevScene S, uint32_t n, float* __restrict__ out, uint32_t* seeds, int shadow)
{
  const uint32_t stride = gridDim.x * blockDim.x;
  for(uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride)
  {
    if(seeds)
      seeds[i] = __float_as_uint(P.misc[i].w);
    if(shadow)
    {
      const float4 c = P.shC[i];
      const bool   occluded = (P.candInfo[i].x & kShadowOccluded) != 0;
      out[i * 3] = occluded ? 0.0f : c.x;
      out[i * 3 + 1] = occluded ? 0.0f : c.y;
      out[i * 3 + 2] = occluded ? 0.0f : c.z;
      continue;
    }
    const float4   h = P.hit[i];
    const uint32_t slot = __float_as_uint(h.w);
    float*         o = out + (size_t)i * 6;
    int            rnode = -1, rprim = -1, primId = -1;
    float          t = kInfinite, u = 0.f, v = 0.f;
    if(slot != 0xFFFFFFFFu)
    {
      const uint2 meta = S.triMeta[slot];
      rnode = (int)(meta.x & 0x0fffffffu);
      rprim = S.nodes[rnode].renderPrimID;
      primId = (int)meta.y;
      t = h.x;
      u = h.y;
      v = h.z;
    }
    o[0] = t;
    o[1] = __int_as_float(rnode);
    o[2] = __int_as_float(rprim);
    o[3] = __int_as_float(primId);
    o[4] = u;
    o[5] = v;
  }
}

// hit-state unit-test hook: the closest hit of a traced ray through k_shade's hit fetch, footprint and material evaluation
// (layout in vk_gltf_renderer_b200/shade_io.py)
PT_D void putShadeField(float* q, int at, float3 v)
{
  q[at] = v.x;
  q[at + 1] = v.y;
  q[at + 2] = v.z;
}
template <uint32_t FEAT>
__global__ void __launch_bounds__(128) k_shade_state(PathState P, DevScene S, const float* __restrict__ in, uint32_t n, float* __restrict__ out, uint32_t* seeds)
{
  stageSrgbLut(S.lutSrgb);
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i >= n)
    return;
  if(seeds)
    seeds[i] = __float_as_uint(P.misc[i].w);
  const float*   p = in + (size_t)i * 16;
  float*         q = out + (size_t)i * 96;
  const float4   hr = P.hit[i];
  const uint32_t slot = __float_as_uint(hr.w);
  for(int k = 0; k < 96; k++)
    q[k] = 0.0f;
  if(slot == 0xFFFFFFFFu)
  {
    q[0] = kInfinite;
    q[1] = q[2] = q[3] = -1.0f;
    return;
  }
  const float3              dir = f3(p[4], p[5], p[6]);
  uint2                     meta;
  const b200pt_render_node* nodeP;
  const HitState            hit = fetchHitState(S, slot, hr.y, hr.z, dir, meta, nodeP);
  const float               worldFoot = rayConeWorldFootprint(p[9], p[10], hr.x, hit.geonrm, dir);
  const float               texGrad = footprintTexGrad(worldFoot, hit.texelDensity, p[11]);
  const PbrMaterial         m = evaluateMaterial<FEAT>(S, S.mats[max(0, nodeP->materialID)], hit, p[8] != 0.0f, texGrad);
  q[0] = hr.x;
  q[1] = (float)(meta.x & 0x0fffffffu);
  q[2] = (float)nodeP->renderPrimID;
  q[3] = (float)meta.y;
  q[4] = hr.y;
  q[5] = hr.z;
  putShadeField(q, 6, hit.pos);
  putShadeField(q, 9, hit.nrm);
  q[12] = hit.color.x;
  q[13] = hit.color.y;
  q[14] = hit.color.z;
  q[15] = hit.color.w;
  putShadeField(q, 16, hit.geonrm);
  putShadeField(q, 19, hit.shadowPos);
  q[22] = hit.uv0.x;
  q[23] = hit.uv0.y;
  q[24] = hit.uv1.x;
  q[25] = hit.uv1.y;
  putShadeField(q, 26, hit.tangent);
  putShadeField(q, 29, hit.bitangent);
  q[32] = hit.texelDensity;
  q[33] = texGrad;
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

// packing of the BSDF test records: vk_gltf_renderer_b200/bsdf_io.py
__device__ PbrMaterial unpackTestMaterial(const float* p)
{
  PbrMaterial m;
  m.baseColor = f3(p[0], p[1], p[2]);
  m.opacity = 1.0f;
  m.roughness = f2(p[3], p[4]);
  m.metallic = p[5];
  m.emissive = f3(0.0f);
  m.N = f3(p[6], p[7], p[8]);
  m.T = f3(p[9], p[10], p[11]);
  m.B = f3(p[12], p[13], p[14]);
  m.Ng = f3(p[15], p[16], p[17]);
  m.ior1 = p[18];
  m.ior2 = p[19];
  m.specular = p[20];
  m.specularColor = f3(p[21], p[22], p[23]);
  m.transmission = p[24];
  m.attenuationColor = f3(1.0f);
  m.attenuationDistance = 1.0f;
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
  m.scatterCoefficient = f3(0.0f);
  m.scatterAnisotropy = 0.0f;
  m.dispersion = 0.0f;
  m.retroreflection = 0.0f;
  return m;
}

__global__ void k_bsdf_eval(const float* __restrict__ in, uint32_t n, float* __restrict__ out)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i >= n)
    return;
  const float*      p = in + (size_t)i * 48;
  const PbrMaterial m = unpackTestMaterial(p);
  const BsdfEval    d = bsdfEvaluate<FEAT_ALL>(m, f3(p[39], p[40], p[41]), f3(p[42], p[43], p[44]), f3(p[45], p[46], p[47]));
  float*            q = out + (size_t)i * 8;
  q[0] = d.bsdf_diffuse.x;
  q[1] = d.bsdf_diffuse.y;
  q[2] = d.bsdf_diffuse.z;
  q[3] = d.bsdf_glossy.x;
  q[4] = d.bsdf_glossy.y;
  q[5] = d.bsdf_glossy.z;
  q[6] = d.pdf;
  q[7] = 0.f;
}

__global__ void k_bsdf_sample(const float* __restrict__ in, uint32_t n, float* __restrict__ out)
{
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i >= n)
    return;
  const float*      p = in + (size_t)i * 48;
  const PbrMaterial m = unpackTestMaterial(p);
  const BsdfSample  d = bsdfSample<FEAT_ALL>(m, f3(p[39], p[40], p[41]), f3(p[45], p[46], p[47]));
  float*            q = out + (size_t)i * 8;
  q[0] = d.k2.x;
  q[1] = d.k2.y;
  q[2] = d.k2.z;
  q[3] = d.bsdf_over_pdf.x;
  q[4] = d.bsdf_over_pdf.y;
  q[5] = d.bsdf_over_pdf.z;
  q[6] = d.pdf;
  q[7] = (float)d.event_type;
}

// texture unit-test hook: one production lookup per record (layout in vk_gltf_renderer_b200/tex_io.py) --
// mode 0 the shade path's getTexture, mode 1 the generic alpha test's sampleLevel0 on the selected texture coordinate
__global__ void k_texture_lookup(DevScene S, const float* __restrict__ in, uint32_t n, float* __restrict__ out)
{
  stageSrgbLut(S.lutSrgb);
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if(i >= n)
    return;
  const float*   p = in + (size_t)i * 8;
  const uint16_t slot = (uint16_t)p[0];
  const float2   tc0 = f2(p[2], p[3]), tc1 = f2(p[4], p[5]);
  float4         r;
  if(p[1] == 0.0f)
    r = getTexture(S, slot, tc0, tc1, p[6]);
  else
  {
    const b200pt_texture_info ti = S.texInfos[slot];
    r = sampleLevel0(S, ti, ti.texCoord ? tc1 : tc0);
  }
  float* q = out + (size_t)i * 4;
  q[0] = r.x;
  q[1] = r.y;
  q[2] = r.z;
  q[3] = r.w;
}

// -------------------------------------------------------------------------------------------------
// host side
// -------------------------------------------------------------------------------------------------

// Owner of the device allocations of one lifetime (the handle, a scene, a path pool, ...): they are freed together, by release() or
// the destructor.  A call that fails returns nullptr and clears the CUDA error; the arena keeps the first failure for the caller's
// report (`failed`), so a step may check once after several allocations.
class DeviceArena
{
public:
  DeviceArena() = default;
  DeviceArena(const DeviceArena&) = delete;
  DeviceArena& operator=(const DeviceArena&) = delete;
  DeviceArena(DeviceArena&& o) noexcept : ptrs(std::move(o.ptrs)), error(o.error) { o.ptrs.clear(); }
  DeviceArena& operator=(DeviceArena&& o) noexcept
  {
    release();
    ptrs.swap(o.ptrs);
    std::swap(error, o.error);
    return *this;
  }
  ~DeviceArena() { release(); }

  // n elements; at least one, so that every buffer has an address
  template <typename T>
  T* alloc(size_t n)
  {
    void* p = nullptr;
    if(!keep(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T))))
      return nullptr;
    ptrs.push_back(p);
    return static_cast<T*>(p);
  }
  // n elements copied from the host on `stream`; n == 0 gives one zeroed element
  template <typename T>
  T* upload(const T* src, size_t n, cudaStream_t stream)
  {
    T* d = alloc<T>(n);
    if(d && !keep(n ? cudaMemcpyAsync(d, src, n * sizeof(T), cudaMemcpyHostToDevice, stream) : cudaMemsetAsync(d, 0, sizeof(T), stream)))
      return nullptr;
    return d;
  }
  void release()
  {
    for(void* p : ptrs)
      cudaFree(p);
    ptrs.clear();
    error = cudaSuccess;
  }
  bool        ok() const { return error == cudaSuccess; }
  cudaError_t takeError() { return std::exchange(error, cudaSuccess); }

private:
  bool keep(cudaError_t e)
  {
    if(e == cudaSuccess)
      return true;
    cudaGetLastError();
    if(error == cudaSuccess)
      error = e;
    return false;
  }
  std::vector<void*> ptrs;
  cudaError_t        error = cudaSuccess;
};

}  // namespace

struct b200pt
{
  int          device = 0;
  cudaStream_t stream = nullptr;
  std::string  err;
  int          numSMs = 132;  // H100 SXM; b200pt_create reads the device's count
  DeviceArena  mem;           // dStats, dLutSrgb, dTmHist and the lanes' counters and buckets

  // scene
  DeviceArena         sceneMem;  // what b200pt_set_scene uploads that no scene edit replaces, and dPrevO2W
  DeviceArena         treeMem;   // the trees and every per-slot table over them: what a rebuild after a scene edit replaces
  DeviceArena         tableMem;  // S.mats and S.texInfos (b200pt_update_materials replaces them)
  DeviceArena         lightMem;  // S.lights (b200pt_update_lights)
  // host copies of what the scene edits compare against or rebuild from
  std::vector<b200pt_shade_material> materials;
  std::vector<b200pt_texture_info>   texInfos;
  std::vector<uint8_t>               visible;    // per render node
  std::vector<DevTex>                devTex;     // S.textures ...
  std::vector<const uchar4*>         texLevel0;  // ... and their level-0 texels
  AlphaRec*                          dAlphaRecsW = nullptr;  // == S.alphaRecs, writable
  uint32_t*                          dMatOfSlotW = nullptr;  // == S.matOfSlot, writable
  const void*         treeBase = nullptr;  // the trees' node + triangle arrays (one allocation) and their size: the L2 window
  size_t              treeBytes = 0;
  // opacity micromaps as handed over by b200pt_set_opacity_micromaps (host copies; consumed by the next b200pt_set_scene)
  struct OmmHost
  {
    std::vector<uint8_t>                  data;
    std::vector<b200pt_micromap_triangle> tris;
  };
  struct PrimOmmHost
  {
    uint32_t             prim = 0, micromap = 0, base = 0;
    bool                 hasIdx = false;
    std::vector<int32_t> idx;
  };
  std::vector<OmmHost>     omms;
  std::vector<PrimOmmHost> primOmms;
  uint32_t                 ommTriangles = 0;  // non-opaque triangles of the scene that got a micromap / special state
  DeviceArena              capMem;            // the alpha caps (alpha_caps.cuh), baked again after every change of the alpha records
  DevScene            S{};
  bool                haveScene = false;
  uint32_t            numTextureInfos = 0;  // S.texInfos entries (host copy of the count, for argument checks)
  bool                hasVolume = false;
  int                 bvhBuilder = 0;  // 0: host SAH builder (bvh.cpp), 1: device LBVH (lbvh.cuh); b200pt_set_bvh_builder
  double              bvhBuildMs = 0.0;  // wall time of the last scene's tree builds
  // any-hit continuation rounds per bounce (B200PT_CONT_ROUNDS, 1..kContRoundsMax).  With one round the in-kernel fallback walks of the
  // last k_alpha (2 of 32 lanes busy) are a tail on every bounce; more rounds move that work into full-width walk launches.
  int                 contRounds = 2;
  // grids of the continuation rounds after the first: -1 = by wavefront size (quarter-size grids below 8 M path slots), 0 = always full,
  // 1 = always quarter-size (B200PT_CONT_SMALL_GRID).  On a small wavefront (a multi-GPU tile) an almost empty full-size walk launch
  // costs about as much as the round saves in k_alpha, hence quarter-size grids there.
  int                 contSmallGrid = -1;
  bool                sortShade = false;  // B200PT_SORT_SHADE=1: material-sorted shade queue
  bool                leanShade = false;  // scene fits the FEAT_LEAN shade variant (scene_feature_detection analogue)
  uint32_t            featureMask = 0;
  uint64_t            nodeBytes = 0, triBytes = 0;
  uint32_t            numNodes = 0, numTris = 0;
  // writable views of the trees for b200pt_update_transforms (refit): [0] merged, [1] opaque-only, [2] non-opaque
  struct TreeDev
  {
    float*                                     nodes = nullptr;
    float*                                     tris = nullptr;   // the triangle array the tree indexes ([1] and [2] share one)
    uint2*                                     meta = nullptr;
    float4*                                    nodeBox = nullptr;  // 2 per node: world-space box (refit scratch)
    uint32_t                                   numNodes = 0, numTriSlots = 0;
    std::vector<std::pair<uint32_t, uint32_t>> levels;  // (first node, count) per depth: builders emit breadth first
  };
  TreeDev             tree[3];
  uint32_t            numSceneNodes = 0;
  b200pt_render_node* dNodesW = nullptr;  // == S.nodes, writable
  const DevPrim*      dPrimsW = nullptr;
  // animation feed (b200pt_set_animation / b200pt_animate): host copy of every primitive's device arrays + sizes, the writable
  // shade records, the uploaded static task inputs and the per-frame buffers (m_morphWeightsBuffer / m_jointMatricesBuffer /
  // m_normalMatricesBuffer of SceneAnimationVk, with per-task offsets)
  struct PrimHost
  {
    DevPrim  d{};
    uint32_t vertexCount = 0, triCount = 0, recBase = 0;
  };
  std::vector<PrimHost>     primHost;
  ShadeRec*                 dShadeRecsW = nullptr;
  struct Animation
  {
    DeviceArena               mem;
    std::vector<MorphTaskDev> morphTasks;
    std::vector<SkinTaskDev>  skinTasks;
    std::vector<uint32_t>     morphPrim, skinPrim;  // renderPrimID per task
    float *                   dMorphWeights = nullptr, *dJointMats = nullptr, *dNormalMats = nullptr;
    size_t                    numMorphWeights = 0, numJoints = 0;
  };
  Animation anim;
  // node hierarchy on the device (b200pt_set_node_hierarchy / b200pt_update_node_matrices)
  struct Hierarchy
  {
    DeviceArena           mem;
    std::vector<uint32_t> levelOffsets;
    uint32_t              numGraphNodes = 0;
    int *                 dParents = nullptr, *dTopo = nullptr;
    float *               dLocalMats = nullptr, *dWorldMats = nullptr, *dInstLocal = nullptr;
    RenderNodeMapping*    dMappings = nullptr;
  };
  Hierarchy graph;

  // env (S.envRgba / S.envAccel point into envMem)
  DeviceArena envMem;
  bool        haveEnv = false;

  // framebuffer + path pool
  int                width = 0, height = 0, tileY0 = 0, tileRows = 0;
  int                bandRows = 0, bandWorld = 1, bandRank = 0;
  uint32_t           numPaths = 0;
  float4*            dAccumOwned = nullptr;
  float4*            dAccum = nullptr;
  bool               guides = false;      // b200pt_set_guide_outputs: the path pools carry guideA / guideN, dGuide is the eOptixAlbedoNormal image
  float4*            dGuide = nullptr;
  // b200pt_set_dlss_guides: the path pools carry guideA / guideN + prevHit / dlssSpec, dDlss holds the six guide planes (28 B per pixel)
  bool               dlss = false;
  uint8_t*           dDlss = nullptr;
  // previous-frame objectToWorld of every render node (k_snapshot_prev_transforms): taken by the first transform update after a
  // rendered frame, read by the next frame only
  float*             dPrevO2W = nullptr;
  bool               prevO2WValid = false;
  bool               renderedSinceUpdate = false;
  uchar4*            dTonemapped = nullptr;  // gBuffers[eImgTonemapped] of this tile (b200pt_tonemap), in poolMem
  uint32_t*          dTmHist = nullptr;      // 256-bin log2-luminance histogram + the exposure factor behind it (allocated with the handle)
  uint32_t*          dSelect = nullptr;  // frame-0 outputs (gltf_pathtrace.slang:610-616): object id per pixel ...
  float*             dNdcDepth = nullptr;  // ... and NDC depth of the first hit
  // Frames in flight (like the reference app's swapchain ring): every lane owns a stream, a path pool, queues and
  // counters; frame f runs its bounces on lane f % numLanes and only k_accumulate runs on the main stream, in
  // frame order.  The latency-bound tail of frame f (a few deep paths) overlaps the wide first bounces of f+1.
  struct Lane
  {
    cudaStream_t stream = nullptr;
    PathState    P{};
    uint32_t*    dQ[6] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};  // trace ping/pong, post, shadow, alpha, continuation
    uint32_t*    dCounters = nullptr;
    uint32_t*    dBuckets = nullptr;  // material-sorted shade queue: [0..1023] bucket counts, [1024..2047] bucket cursors
    uint32_t*    hCount = nullptr;   // pinned
    cudaEvent_t  done = nullptr;     // lane stream: all bounces of the lane's frame enqueued before it
    cudaEvent_t  freed = nullptr;    // main stream: k_accumulate has consumed the lane's pixSum
    bool         busy = false;       // `freed` has been recorded at least once since the pool was (re)built
    ViewPose*    poses = nullptr;    // views > 1: the poses of the lane's frame (FrameParams::poses)
  };
  static constexpr int kMaxLanes = 8;
  Lane               lanes[kMaxLanes];
  // frame batching (b200pt_set_frame_batch): up to `batch` consecutive frames of a static camera are collected and run as one
  // wavefront of batch x pixels paths (a multi-GPU tile is 1/N of the frame: batching N frames gives its kernels the size of a
  // single-GPU frame and divides the launches per frame by N)
  int                   batch = 1;
  int                   pendingCount = 0;
  b200pt_frame_info     pendingFi{};
  b200pt_push_constant  pendingPc{};  // the FIRST pending frame's constants
  // views (b200pt_set_views / b200pt_render_views): `views` camera poses of one frame run as one wavefront of views x pixels paths,
  // each into its own images.  View 0 is dAccum / dSelect / dNdcDepth; views 1.. are (views - 1) x pixels images in poolMem.
  int                   views = 1;
  float4*               dViewAccum = nullptr;
  uint32_t*             dViewSelect = nullptr;
  float*                dViewDepth = nullptr;
  int                numLanes = 4;   // frames in flight (b200pt_set_frames_in_flight)
  uint64_t           frameSerial = 0;
  int                lastLane = -1;
  cudaEvent_t        readDone[8] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  DeviceArena        poolMem;
  // scratch pool of the ray-level API (b200pt_trace_closest / b200pt_trace_shadow run the production kernels on it)
  PathState          rayP{};
  uint32_t*          rayQ[3] = {nullptr, nullptr, nullptr};  // rays, any-hit, continuation
  uint32_t*          rayCounters = nullptr;                  // one iteration of the Counters layout
  uint32_t           rayCapacity = 0;
  DeviceArena        rayMem;
  DevStats*          dStats = nullptr;
  float*             dLutSrgb = nullptr;

  // stats / profiling: CUDA-event pairs recorded around every launch on the handle's stream and
  // resolved lazily (no host sync inside a frame)
  struct EvRec
  {
    cudaEvent_t a, b;
    Stage       cat;
    int         lane;  // timeline: stream the launch went to (-1 main)
    uint64_t    frame;
    int         bounce;  // -1 outside the bounce loop
  };
  bool               profiling = false;
  // B200PT_TIMELINE=<file>: event pairs around every launch WITHOUT serialising the frames in flight; flushEvents appends
  // "frame,lane,stage,start_ms,end_ms" rows (times relative to tlBase) -- the per-rank timeline of a real run
  FILE*              timeline = nullptr;
  cudaEvent_t        tlBase = nullptr;
  std::vector<EvRec> evPool;
  size_t             evUsed = 0;
  double             msCat[kStageCount] = {};
  uint64_t           launchesCat[kStageCount] = {};
  uint64_t           kernelLaunches = 0;
};

namespace {

#define CK(call)                                                                                                                            \
  do                                                                                                                                        \
  {                                                                                                                                         \
    cudaError_t e__ = (call);                                                                                                               \
    if(e__ != cudaSuccess)                                                                                                                  \
    {                                                                                                                                       \
      h->err = std::string(#call) + ": " + cudaGetErrorString(e__);                                                                         \
      return B200PT_E_CUDA;                                                                                                                 \
    }                                                                                                                                       \
  } while(0)

// the exit of a step whose arena failed: B200PT_E_NOMEM when the device is out of memory, B200PT_E_CUDA for any other error;
// `what` names the buffer
int failed(b200pt* h, DeviceArena& A, const char* what)
{
  const cudaError_t e = A.takeError();
  if(e == cudaErrorMemoryAllocation)
  {
    h->err = std::string(what) + ": out of device memory";
    return B200PT_E_NOMEM;
  }
  h->err = std::string(what) + ": " + cudaGetErrorString(e);
  return B200PT_E_CUDA;
}

// the SoA arrays of one path pool (device_scene.cuh: PathState) for n paths; the caller checks A
void allocPathState(const b200pt* h, DeviceArena& A, size_t n, PathState& P)
{
  P = PathState{};
  float4** arrays[] = {&P.rayO, &P.rayD, &P.hit, &P.thr, &P.rad, &P.misc, reinterpret_cast<float4**>(&P.medium), &P.pixSum, &P.shO, &P.shD, &P.shC, &P.firstHit};
  for(float4** a : arrays)
    *a = A.alloc<float4>(n);
  for(int k = 0; k < kCand; k++)
    P.cand[k] = A.alloc<float4>(n);
  P.candInfo = A.alloc<uint2>(n);
  if(h->guides || h->dlss)
  {
    P.guideA = A.alloc<float4>(n);
    P.guideN = A.alloc<float4>(n);
  }
  if(h->dlss)
  {
    P.prevHit = A.alloc<float4>(n);
    P.dlssSpec = A.alloc<uint2>(n);
  }
}

// Builds one compressed wide BVH over `m` of the scene's triangles ON THE DEVICE (lbvh.cuh) and brings it back in the host
// builder's format, so that everything downstream of the builders (uploads, record tables, refit levels) is shared.
// dInRec: 12 floats per global triangle in flatten order; dSubset: m global ids or nullptr.
int buildWideBvhGpu(b200pt* h, const float* dInRec, const uint32_t* dSubset, uint32_t m, uint32_t triBaseOffset, WideBvh& out)
{
  out = WideBvh();
  out.numTris = m;
  if(m == 0)
  {
    out.nodes.assign(20, 0.f);
    out.numNodes = 1;
    return B200PT_OK;
  }
  uint32_t M = 1;
  while(M < m)
    M <<= 1;
  DeviceArena A;  // the build's scratch, freed on every return
  auto        cudaFailed = [&]() {
    h->err = "GPU BVH build failed (launch or copy)";
    return B200PT_E_CUDA;
  };
  LbvhWork W{};
  W.m = m;
  W.M = M;
  W.inRec = dInRec;
  W.subset = dSubset;
  W.triBaseOffset = triBaseOffset;
  W.primLo = A.alloc<float4>(m);
  W.primHi = A.alloc<float4>(m);
  W.keys = A.alloc<unsigned long long>(M);
  W.left = A.alloc<int>(m);
  W.right = A.alloc<int>(m);
  W.parentI = A.alloc<int>(m);
  W.parentL = A.alloc<int>(m);
  W.first = A.alloc<uint32_t>(m);
  W.last = A.alloc<uint32_t>(m);
  W.boxLo = A.alloc<float4>(m);
  W.boxHi = A.alloc<float4>(m);
  W.visits = A.alloc<uint32_t>(m);
  W.cbounds = A.alloc<int>(6);
  W.nodes = A.alloc<float>(((size_t)m + 1) * 20);
  W.tris = A.alloc<float>((size_t)m * 12);
  W.triMeta = A.alloc<uint32_t>((size_t)m * 2);
  W.counters = A.alloc<uint32_t>(4);
  int2* queue[2] = {A.alloc<int2>((size_t)m + 1), A.alloc<int2>((size_t)m + 1)};
  if(!A.ok())
    return failed(h, A, "GPU BVH build");
  cudaStream_t st = h->stream;
  const int    cbInit[6] = {0x7fffffff, 0x7fffffff, 0x7fffffff, (int)0x80000000, (int)0x80000000, (int)0x80000000};
  const uint32_t cnt0[4] = {1u, 0u, 0u, 0u};  // wide node 0 is the root
  bool         ok = cudaMemcpyAsync(W.cbounds, cbInit, sizeof(cbInit), cudaMemcpyHostToDevice, st) == cudaSuccess;
  ok = ok && cudaMemcpyAsync(W.counters, cnt0, sizeof(cnt0), cudaMemcpyHostToDevice, st) == cudaSuccess;
  ok = ok && cudaMemsetAsync(W.visits, 0, (size_t)m * 4, st) == cudaSuccess;
  ok = ok && cudaMemsetAsync(W.nodes, 0, ((size_t)m + 1) * 80, st) == cudaSuccess;
  if(!ok)
    return cudaFailed();
  const uint32_t gm = (m + 255) / 256, gM = (M + 255) / 256;
  k_lbvh_bounds<<<gm, 256, 0, st>>>(W);
  k_lbvh_morton<<<gM, 256, 0, st>>>(W);
  for(uint32_t k = 2; k <= M; k <<= 1)
    for(uint32_t j = k >> 1; j > 0; j >>= 1)
      k_lbvh_bitonic<<<gM, 256, 0, st>>>(W.keys, M, j, k);
  if(m >= 2)
  {
    k_lbvh_hierarchy<<<gm, 256, 0, st>>>(W);
    k_lbvh_fit<<<gm, 256, 0, st>>>(W);
  }
  h->kernelLaunches += 4;
  // collapse + emit, level by level
  const int2 rootEntry = make_int2(m >= 2 ? 0 : ~0, 0);
  if(cudaMemcpyAsync(queue[0], &rootEntry, sizeof(rootEntry), cudaMemcpyHostToDevice, st) != cudaSuccess)
    return cudaFailed();
  uint32_t count = 1, depth = 0;
  int      cur = 0;
  while(count)
  {
    const uint32_t zero = 0;
    if(cudaMemcpyAsync(&W.counters[2], &zero, 4, cudaMemcpyHostToDevice, st) != cudaSuccess)
      return cudaFailed();
    k_lbvh_emit<<<(count + 127) / 128, 128, 0, st>>>(W, queue[cur], count, queue[1 - cur]);
    h->kernelLaunches++;
    if(cudaMemcpyAsync(&count, &W.counters[2], 4, cudaMemcpyDeviceToHost, st) != cudaSuccess || cudaStreamSynchronize(st) != cudaSuccess)
      return cudaFailed();
    cur = 1 - cur;
    depth++;
    if(depth > 64)
      return cudaFailed();
  }
  uint32_t cnt[2] = {0, 0};
  if(cudaMemcpy(cnt, W.counters, 8, cudaMemcpyDeviceToHost) != cudaSuccess || cnt[1] != m || cnt[0] == 0 || cnt[0] > m + 1)
    return cudaFailed();
  out.numNodes = cnt[0];
  out.maxDepth = depth;
  out.nodes.resize((size_t)cnt[0] * 20);
  out.tris.resize((size_t)m * 12);
  out.triMeta.resize((size_t)m * 2);
  if(cudaMemcpy(out.nodes.data(), W.nodes, out.nodes.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess
     || cudaMemcpy(out.tris.data(), W.tris, out.tris.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess
     || cudaMemcpy(out.triMeta.data(), W.triMeta, out.triMeta.size() * 4, cudaMemcpyDeviceToHost) != cudaSuccess)
    return cudaFailed();
  return B200PT_OK;
}

void freeRayPool(b200pt* h)
{
  h->rayMem.release();
  h->rayCapacity = 0;
}

// drops the scene and everything built on it; h->S keeps only the environment and the sRGB table, h->tree[] is empty
void freeScene(b200pt* h)
{
  h->dPrevO2W = nullptr;
  h->prevO2WValid = false;
  h->renderedSinceUpdate = false;
  h->anim = b200pt::Animation{};
  h->graph = b200pt::Hierarchy{};
  h->treeMem.release();
  h->capMem.release();
  h->tableMem.release();
  h->lightMem.release();
  h->sceneMem.release();
  h->primHost.clear();
  h->materials.clear();
  h->texInfos.clear();
  h->visible.clear();
  h->devTex.clear();
  h->texLevel0.clear();
  h->dAlphaRecsW = nullptr;
  h->dMatOfSlotW = nullptr;
  h->dShadeRecsW = nullptr;
  h->dNodesW = nullptr;
  h->dPrimsW = nullptr;
  h->numSceneNodes = 0;
  for(auto& t : h->tree)
    t = b200pt::TreeDev();
  const DevScene old = h->S;
  h->S = DevScene{};
  h->S.envRgba = old.envRgba;
  h->S.envAccel = old.envAccel;
  h->S.envW = old.envW;
  h->S.envH = old.envH;
  h->S.lutSrgb = h->dLutSrgb;
  h->haveScene = false;
}

void syncAll(b200pt* h)
{
  for(int l = 0; l < b200pt::kMaxLanes; l++)
    if(h->lanes[l].stream)
      cudaStreamSynchronize(h->lanes[l].stream);
  cudaStreamSynchronize(h->stream);
}

void freePool(b200pt* h)
{
  for(int l = 0; l < b200pt::kMaxLanes; l++)
    h->lanes[l].busy = false;
  h->lastLane = -1;
  h->poolMem.release();
  h->dAccumOwned = nullptr;
  h->dAccum = nullptr;
  h->dSelect = nullptr;
  h->dNdcDepth = nullptr;
  h->dTonemapped = nullptr;
  h->dGuide = nullptr;
  h->dDlss = nullptr;
  h->dViewAccum = nullptr;
  h->dViewSelect = nullptr;
  h->dViewDepth = nullptr;
  h->numPaths = 0;
  for(int l = 0; l < b200pt::kMaxLanes; l++)
  {
    h->lanes[l].P = PathState{};
    h->lanes[l].poses = nullptr;
    for(int k = 0; k < 6; k++)
      h->lanes[l].dQ[k] = nullptr;
  }
}

void flushEvents(b200pt* h)
{
  if(h->evUsed == 0)
    return;
  syncAll(h);
  for(size_t i = 0; i < h->evUsed; i++)
  {
    float ms = 0.f;
    if(cudaEventElapsedTime(&ms, h->evPool[i].a, h->evPool[i].b) == cudaSuccess)
    {
      h->msCat[h->evPool[i].cat] += ms;
      h->launchesCat[h->evPool[i].cat]++;
    }
    if(h->timeline && h->tlBase)
    {
      float t0 = 0.f, t1 = 0.f;
      if(cudaEventElapsedTime(&t0, h->tlBase, h->evPool[i].a) == cudaSuccess && cudaEventElapsedTime(&t1, h->tlBase, h->evPool[i].b) == cudaSuccess)
        fprintf(h->timeline, "%llu,%d,%s,%.4f,%.4f\n", (unsigned long long)h->evPool[i].frame, h->evPool[i].lane, kStageName[h->evPool[i].cat], t0, t1);
    }
  }
  if(h->timeline)
    fflush(h->timeline);
  h->evUsed = 0;
}

// grows the pool of profiling event pairs to n entries, up to the first failed cudaEventCreate
cudaError_t growEventPool(b200pt* h, size_t n)
{
  cudaError_t e = cudaSuccess;
  for(size_t i = h->evPool.size(); i < n && e == cudaSuccess; i++)
  {
    h->evPool.emplace_back();
    e = cudaEventCreate(&h->evPool[i].a);
    if(e == cudaSuccess)
      e = cudaEventCreate(&h->evPool[i].b);
  }
  return e;
}

float srgbToLinear(float c) { return (c <= 0.04045f) ? c / 12.92f : powf((c + 0.055f) / 1.055f, 2.4f); }
float linearToSrgb(float c) { return (c <= 0.0031308f) ? c * 12.92f : 1.055f * powf(c, 1.0f / 2.4f) - 0.055f; }

// mip chain like the reference's vkCmdBlitImage(VK_FILTER_LINEAR) loop (src/gltf_scene_vk.cpp:1254-1332):
// every level is the linear-filtered half-size copy of the previous 8-bit level (sRGB images are
// filtered in linear light and re-encoded).
void downsample(const std::vector<uint8_t>& src, int w, int h, bool srgb, std::vector<uint8_t>& dst, int nw, int nh)
{
  dst.resize((size_t)nw * nh * 4);
  std::vector<float> lin((size_t)w * h * 4);
  float              lutL[256], lutS[256];
  for(int i = 0; i < 256; i++)
  {
    lutL[i] = (float)i / 255.0f;
    lutS[i] = srgbToLinear((float)i / 255.0f);
  }
  for(size_t i = 0; i < (size_t)w * h; i++)
    for(int c = 0; c < 4; c++)
      lin[i * 4 + c] = (srgb && c < 3) ? lutS[src[i * 4 + c]] : lutL[src[i * 4 + c]];
  for(int y = 0; y < nh; y++)
    for(int x = 0; x < nw; x++)
    {
      const float sx = (x + 0.5f) * (float)w / (float)nw - 0.5f;
      const float sy = (y + 0.5f) * (float)h / (float)nh - 0.5f;
      int         x0 = (int)floorf(sx), y0 = (int)floorf(sy);
      const float fx = sx - x0, fy = sy - y0;
      const int   x1 = std::min(x0 + 1, w - 1), y1 = std::min(y0 + 1, h - 1);
      x0 = std::max(x0, 0);
      y0 = std::max(y0, 0);
      for(int c = 0; c < 4; c++)
      {
        const float a = lin[((size_t)y0 * w + x0) * 4 + c], b = lin[((size_t)y0 * w + x1) * 4 + c];
        const float cc = lin[((size_t)y1 * w + x0) * 4 + c], d = lin[((size_t)y1 * w + x1) * 4 + c];
        float       v = (a * (1 - fx) + b * fx) * (1 - fy) + (cc * (1 - fx) + d * fx) * fy;
        if(srgb && c < 3)
          v = linearToSrgb(v);
        dst[((size_t)y * nw + x) * 4 + c] = (uint8_t)std::min(255.0f, std::max(0.0f, floorf(v * 255.0f + 0.5f)));
      }
    }
}

struct MipChain
{
  std::vector<std::vector<uint8_t>> level;
  std::vector<int>                  w, h;
};

void buildMipChain(const b200pt_texture& src, MipChain& mc)
{
  int w = src.width, hh = src.height;
  mc.level.emplace_back(src.rgba8, src.rgba8 + (size_t)w * hh * 4);
  mc.w.push_back(w);
  mc.h.push_back(hh);
  while(w > 1 || hh > 1)
  {
    const int            nw = std::max(1, w / 2), nh = std::max(1, hh / 2);
    std::vector<uint8_t> nxt;
    downsample(mc.level.back(), w, hh, src.srgb != 0, nxt, nw, nh);
    mc.level.push_back(std::move(nxt));
    mc.w.push_back(nw);
    mc.h.push_back(nh);
    w = nw;
    hh = nh;
  }
}

// texels of one mip chain in the device layout: level after level, each as row-major 4x4-texel tiles
// (levels narrower than 4 texels are padded; the padding is never addressed)
void packTiled(const MipChain& mc, std::vector<uint32_t>& texels, uint32_t levelOfs[16])
{
  for(size_t l = 0; l < mc.level.size() && l < 16; l++)
  {
    const int w = mc.w[l], hh = mc.h[l], tpr = (w + 3) >> 2, tpc = (hh + 3) >> 2;
    levelOfs[l] = (uint32_t)texels.size();
    texels.resize(texels.size() + (size_t)tpr * tpc * 16, 0u);
    uint32_t*       dst = texels.data() + levelOfs[l];
    const uint32_t* src = reinterpret_cast<const uint32_t*>(mc.level[l].data());
    for(int y = 0; y < hh; y++)
      for(int x = 0; x < w; x++)
        dst[(((size_t)(y >> 2) * tpr + (x >> 2)) << 4) + ((y & 3) << 2) + (x & 3)] = src[(size_t)y * w + x];
  }
}

void describeTexture(const b200pt_texture& src, const MipChain& mc, DevTex& dev)
{
  const int levels = (int)std::min<size_t>(mc.level.size(), 16);
  // sampler quirks kept from getSampler (src/gltf_scene_vk.cpp:909-947): the mip mode follows magFilter, and magFilter goes
  // through the same table as minFilter (9728 / 9984 / 9986 are NEAREST)
  const bool magNearest = src.magFilter == 9728 || src.magFilter == 9984 || src.magFilter == 9986;
  dev.w0 = src.width;
  dev.h0 = src.height;
  dev.maxLevel = (float)(levels - 1);
  dev.wrapS = src.wrapS;
  dev.wrapT = src.wrapT;
  dev.srgb = src.srgb ? 1 : 0;
  dev.magLinear = magNearest ? 0 : 1;
  dev.minLinear = (src.minFilter == 9728 || src.minFilter == 9984 || src.minFilter == 9986) ? 0 : 1;
  dev.mipLinear = magNearest ? 0 : 1;
}

int gridFor(const b200pt* h, int perSM) { return h->numSMs * perSM; }

// The launches of one frame or one ray-level call.  Every launch is counted in kernelLaunches; a timed one (a frame while profiling or
// with B200PT_TIMELINE) is wrapped in an event pair tagged with its stage, lane, frame and bounce.
struct Launcher
{
  b200pt*      h;
  cudaStream_t stream;
  int          lane;  // -1: the handle's stream
  uint64_t     frame;
  int          bounce;  // -1 outside the bounce loop
  bool         timed;
  uint32_t     paths;  // path slots of the wavefront
  template <class F>
  void operator()(Stage stage, F&& launch) const
  {
    if(timed)
    {
      if(h->evUsed == h->evPool.size())
        flushEvents(h);
      b200pt::EvRec& r = h->evPool[h->evUsed++];
      r.cat = stage;
      r.lane = lane;
      r.frame = frame;
      r.bounce = bounce;
      cudaEventRecord(r.a, stream);
      launch(stream);
      cudaEventRecord(r.b, stream);
    }
    else
      launch(stream);
    h->kernelLaunches++;
  }
};

// The walk of queue q (closest-hit or shadow rays) with its any-hit rounds through the any-hit and continuation queues qAlpha / qCont:
// walk -> [k_alpha -> continuation walk] x contRounds -> k_alpha in a scene with non-opaque triangles, the bare walk otherwise.
// baseMode is added to every launch's mode (TRACE_TMIN: closest rays of the ray-level API).
void launchWalk(const Launcher& ctx, int shadow, const PathState& P, const uint32_t* q, uint32_t* qAlpha, uint32_t* qCont, const Counters& C, int it,
                int baseMode)
{
  const b200pt*   h = ctx.h;
  const DevScene& S = h->S;
  // the walk kernels have an instantiation for scenes with opacity micromaps (omm.cuh), one for scenes with alpha caps (alpha_caps.cuh)
  // and one without either lookup
  const bool  omm = S.bvh.ommRef != nullptr, caps = S.bvh.capRef != nullptr;
  const auto  walk = shadow ? (omm ? k_shadow<true, false> : caps ? k_shadow<false, true> : k_shadow<false, false>)
                            : (omm ? k_trace<true, false> : caps ? k_trace<false, true> : k_trace<false, false>);
  const auto  alpha = shadow ? k_alpha<true> : k_alpha<false>;
  const Stage stage = shadow ? kStageShadow : kStageTrace;
  const int   gA = gridFor(h, 8), gW = gridFor(h, kWalkCtasPerSM), R = h->contRounds;
  // rounds after the first see the few rays whose candidates were all rejected twice (about 1 % of a bounce); on a small wavefront
  // a quarter-size grid keeps the fixed cost of these extra launches down (see contSmallGrid)
  const bool  small = h->contSmallGrid < 0 ? (ctx.paths < (8u << 20)) : (h->contSmallGrid != 0);
  ctx(stage, [&](cudaStream_t st) {
    walk<<<gW, 128, 0, st>>>(P, S, q, C.queue(shadow, it), C.cursor(shadow, it), qAlpha, C.anyHit(shadow, 0, it), h->dStats, baseMode);
  });
  if(!S.hasAlpha)
    return;
  for(int r = 0; r < R; r++)
  {
    const int gAr = (r && small) ? gridFor(h, 2) : gA, gWr = (r && small) ? gridFor(h, 2) : gW;
    ctx(kStageAnyHit, [&](cudaStream_t st) {
      alpha<<<gAr, 128, 2048, st>>>(P, S, qAlpha, C.anyHit(shadow, r, it), qCont, C.cont(shadow, r, it), h->dStats, baseMode | (r ? TRACE_CONT : 0));
    });
    ctx(stage, [&](cudaStream_t st) {
      walk<<<gWr, 128, 0, st>>>(P, S, qCont, C.cont(shadow, r, it), C.contCursor(shadow, r, it), qAlpha, C.anyHit(shadow, r + 1, it), h->dStats,
                                baseMode | TRACE_CONT);
    });
  }
  ctx(kStageAnyHit, [&](cudaStream_t st) { alpha<<<gA, 128, 2048, st>>>(P, S, qAlpha, C.anyHit(shadow, R, it), nullptr, nullptr, h->dStats, baseMode | TRACE_CONT); });
}

// counting sort of the queue q of a lane by material into qOut: k_sort_count -> k_sort_scan -> k_sort_scatter over nb buckets
void launchSort(const Launcher& ctx, const b200pt::Lane& L, const uint32_t* q, const uint32_t* cnt, uint32_t* qOut, uint32_t nb)
{
  const b200pt* h = ctx.h;
  const int     g = gridFor(h, 4);
  ctx(kStageOther, [&](cudaStream_t st) { k_sort_count<<<g, 256, 0, st>>>(L.P, h->S, q, cnt, L.dBuckets, nb); });
  ctx(kStageOther, [&](cudaStream_t st) { k_sort_scan<<<1, kSortMaxBuckets, 0, st>>>(L.dBuckets, L.dBuckets + kSortMaxBuckets, nb); });
  ctx(kStageOther, [&](cudaStream_t st) { k_sort_scatter<<<g, 256, 0, st>>>(L.P, h->S, q, cnt, L.dBuckets + kSortMaxBuckets, qOut, nb); });
}

}  // namespace
extern "C" {
static int launchFrames(b200pt_t* h, const b200pt_frame_info* fi, const b200pt_push_constant* pc, int count, const b200pt_frame_info* viewFis = nullptr);
static int flushPending(b200pt_t* h);
}
namespace {

// device-side error flags (DevStats::errorFlags) -> error code; the flag stays set until b200pt_reset_stats
int checkDeviceErrors(b200pt* h)
{
  unsigned long long flags = 0;
  if(cudaMemcpy(&flags, &h->dStats->errorFlags, sizeof(flags), cudaMemcpyDeviceToHost) != cudaSuccess)
  {
    h->err = "reading the device error flags failed";
    return B200PT_E_CUDA;
  }
  if(flags & 1ull)
  {
    h->err = "a traversal stack overflowed: the BVH is deeper than the kernels' stack, results are incomplete";
    return B200PT_E_DEVICE;
  }
  return B200PT_OK;
}

// the prologue of the entry points: the handle's device made current, the batched frames still pending launched and, with `sync`,
// every stream idle, so that no frame in flight still reads what the call changes
int enter(b200pt* h, bool sync)
{
  CK(cudaSetDevice(h->device));
  if(const int rc = flushPending(h))
    return rc;
  if(sync)
    syncAll(h);
  return B200PT_OK;
}

}  // namespace

// =================================================================================================
// C ABI
// =================================================================================================
extern "C" {

int b200pt_abi_version(void) { return B200PT_ABI_VERSION; }

int b200pt_create(b200pt_t** out, int cuda_device)
{
  if(!out)
    return B200PT_E_INVALID;
  *out = nullptr;
  int n = 0;
  if(cudaGetDeviceCount(&n) != cudaSuccess || cuda_device < 0 || cuda_device >= n)
    return B200PT_E_CUDA;
  b200pt* h = new b200pt();
  h->device = cuda_device;
  if(cudaSetDevice(cuda_device) != cudaSuccess || cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking) != cudaSuccess)
  {
    delete h;
    return B200PT_E_CUDA;
  }
  if(const char* e = getenv("B200PT_SORT_SHADE"))
    h->sortShade = atoi(e) != 0;
  if(const char* e = getenv("B200PT_CONT_SMALL_GRID"))
    h->contSmallGrid = atoi(e) != 0 ? 1 : 0;
  if(const char* e = getenv("B200PT_CONT_ROUNDS"))
    h->contRounds = std::min(std::max(atoi(e), 1), kContRoundsMax);
  bool ok = true;
  auto need = [&](cudaError_t e) { ok = ok && (e == cudaSuccess); };
  cudaDeviceProp prop{};
  need(cudaGetDeviceProperties(&prop, cuda_device));
  h->numSMs = prop.multiProcessorCount > 0 ? prop.multiProcessorCount : 132;
  h->dStats = h->mem.alloc<DevStats>(1);
  if(h->dStats)
    need(cudaMemset(h->dStats, 0, sizeof(DevStats)));
  if(const char* e = getenv("B200PT_TIMELINE"))
  {
    // one file per process (ranks of a multi-GPU run append their pid)
    const std::string path = std::string(e) + "." + std::to_string((long long)getpid());
    h->timeline = fopen(path.c_str(), "w");
    if(h->timeline)
    {
      fprintf(h->timeline, "frame,lane,stage,start_ms,end_ms\n");
      need(cudaEventCreate(&h->tlBase));
      need(cudaEventRecord(h->tlBase, h->stream));
      need(growEventPool(h, 16384));
    }
  }
  for(int l = 0; l < b200pt::kMaxLanes; l++)
  {
    b200pt::Lane& L = h->lanes[l];
    need(cudaStreamCreateWithFlags(&L.stream, cudaStreamNonBlocking));
    need(cudaEventCreateWithFlags(&L.done, cudaEventDisableTiming));
    need(cudaEventCreateWithFlags(&L.freed, cudaEventDisableTiming));
    L.dCounters = h->mem.alloc<uint32_t>(kCounterArrays * kMaxIters);
    L.dBuckets = h->mem.alloc<uint32_t>(2 * kSortMaxBuckets);
    if(L.dBuckets)
      need(cudaMemset(L.dBuckets, 0, sizeof(uint32_t) * 2 * kSortMaxBuckets));
    need(cudaMallocHost((void**)&L.hCount, sizeof(uint32_t) * 4));
  }
  {
    // [0..255]: sRGB decode; [256..511]: i / 255 (the UNORM decode, tabulated so that texel fetches do no divisions;
    // same IEEE quotient the kernel's own `(float)i / 255.0f` would produce)
    float lutS[512];
    for(int i = 0; i < 256; i++)
    {
      lutS[i] = srgbToLinear((float)i / 255.0f);
      lutS[256 + i] = (float)i / 255.0f;
    }
    h->dLutSrgb = h->mem.alloc<float>(512);
    h->dTmHist = h->mem.alloc<uint32_t>(kTmBins + 1);  // histogram + the exposure factor (a float in the last word)
    if(h->dLutSrgb)
      need(cudaMemcpy(h->dLutSrgb, lutS, sizeof(lutS), cudaMemcpyHostToDevice));
  }
  if(!ok || !h->mem.ok())
  {
    const int rc = h->mem.ok() ? B200PT_E_CUDA : B200PT_E_NOMEM;
    cudaGetLastError();  // clear the sticky-free error state for the next attempt
    b200pt_destroy(h);
    return rc;
  }
  *out = h;
  return B200PT_OK;
}

void b200pt_destroy(b200pt_t* h)
{
  if(!h)
    return;
  cudaSetDevice(h->device);
  syncAll(h);
  flushEvents(h);  // (writes the tail of a B200PT_TIMELINE dump; needs the lane streams alive)
  freeScene(h);
  freePool(h);
  freeRayPool(h);
  for(int k = 0; k < 8; k++)
    if(h->readDone[k])
      cudaEventDestroy(h->readDone[k]);
  for(int l = 0; l < b200pt::kMaxLanes; l++)
  {
    b200pt::Lane& L = h->lanes[l];
    if(L.hCount)
      cudaFreeHost(L.hCount);
    if(L.done)
      cudaEventDestroy(L.done);
    if(L.freed)
      cudaEventDestroy(L.freed);
    if(L.stream)
      cudaStreamDestroy(L.stream);
  }
  for(auto& e : h->evPool)
  {
    cudaEventDestroy(e.a);
    cudaEventDestroy(e.b);
  }
  if(h->tlBase)
    cudaEventDestroy(h->tlBase);
  if(h->timeline)
    fclose(h->timeline);
  cudaStreamDestroy(h->stream);
  delete h;  // (the arenas free the handle's and the environment's buffers)
}

const char* b200pt_last_error(const b200pt_t* h) { return h ? h->err.c_str() : "null handle"; }

void* b200pt_stream(b200pt_t* h) { return h ? (void*)h->stream : nullptr; }

}  // extern "C"
namespace {

// ---- b200pt_set_scene, step by step: validateScene, then steps that can only fail with E_NOMEM / E_CUDA, then commitScene ----

// what b200pt_set_scene builds before it hands the scene to the handle
struct SceneBuild
{
  DeviceArena                   mem, treeMem, tableMem, lightMem;  // the handle's arenas of the same names (sceneMem = mem)
  DevScene                      S{};
  b200pt_render_node*           nodesW = nullptr;  // == S.nodes, writable
  ShadeRec*                     shadeRecsW = nullptr;  // == S.shadeRecs, writable
  AlphaRec*                     alphaRecsW = nullptr;  // == S.alphaRecs, writable
  uint32_t*                     matOfSlotW = nullptr;  // == S.matOfSlot, writable
  std::vector<b200pt::PrimHost> primHost;
  std::vector<DevTex>           devTex;     // host copies of the texture records ...
  std::vector<const uchar4*>    texLevel0;  // ... and their level-0 texels (device), for the alpha-triangle records
  std::vector<FlatTri>          flat;
  bool                          anyNonOpaque = false;
  WideBvh                       bvh, bvhO, bvhA;
  double                        bvhBuildMs = 0.0;
  const void*                   treeBase = nullptr;
  size_t                        treeBytes = 0;
  b200pt::TreeDev               tree[3];
  uint64_t                      nodeBytes = 0, triBytes = 0;
  uint32_t                      ommTriangles = 0;
};

// the checks of a material table against a texture-info table of numTextureInfos entries (b200pt_set_scene and
// b200pt_update_materials; `who` names the call in the message)
int validateMaterials(b200pt* h, const char* who, const b200pt_shade_material* mats, uint32_t numMaterials, uint32_t numTextureInfos)
{
  for(uint32_t i = 0; i < numMaterials; i++)
  {
    const b200pt_shade_material& m = mats[i];
    // the 22 texture slots index GltfTextureInfo[] (0 = none, shaders/gltf_scene_io.h.slang:196-219)
    const uint16_t* slots = &m.pbrBaseColorTexture;
    for(int k = 0; k < 22; k++)
      if(slots[k] != 0 && slots[k] >= numTextureInfos)
      {
        h->err = std::string(who) + ": material texture slot beyond numTextureInfos";
        return B200PT_E_INVALID;
      }
    if(m.retroreflectionFactor > 0.0f)
    {
      h->err = std::string(who) + ": KHR_materials_retroreflection is not built (its lobe lives in nvshaders, external to the reference tree)";
      return B200PT_E_UNSUPPORTED;
    }
  }
  return B200PT_OK;
}

// a visible render node whose material puts its triangles into the any-hit path exists (render nodes already checked)
bool anyNonOpaqueOf(const b200pt_scene_desc& s)
{
  for(uint32_t n = 0; n < s.numRenderNodes; n++)
  {
    const b200pt_render_node& node = s.renderNodes[n];
    if((!s.renderNodeVisible || s.renderNodeVisible[n]) && s.renderPrimitives[node.renderPrimID].triangleCount
       && !(triFlags(s.materials[materialOf(node)]) & TRI_OPAQUE))
      return true;
  }
  return false;
}

// the micromaps are linked only into scenes with non-opaque triangles (linkMicromaps): then every linked primitive must be covered
int validateMicromaps(b200pt* h, const char* who, const b200pt_scene_desc& s)
{
  if(!anyNonOpaqueOf(s))
    return B200PT_OK;
  for(const auto& po : h->primOmms)
  {
    if(po.prim >= s.numRenderPrimitives)
    {
      h->err = std::string(who) + ": opacity micromap linked to a render primitive out of range";
      return B200PT_E_INVALID;
    }
    const uint32_t nTri = s.renderPrimitives[po.prim].triangleCount;
    if(po.hasIdx ? po.idx.size() < nTri : (uint64_t)po.base + nTri > h->omms[po.micromap].tris.size())
    {
      h->err = std::string(who) + ": opacity micromap does not cover its primitive's triangles";
      return B200PT_E_INVALID;
    }
  }
  return B200PT_OK;
}

// every check of b200pt_set_scene, before its first allocation
int validateScene(b200pt* h, const b200pt_scene_desc& s)
{
  auto refuse = [&](const std::string& msg) {
    h->err = msg;
    return B200PT_E_INVALID;
  };
  if(const int rc = validateMaterials(h, "b200pt_set_scene", s.materials, s.numMaterials, s.numTextureInfos))
    return rc;
  for(uint32_t i = 0; i < s.numTextures; i++)
  {
    const b200pt_texture& t = s.textures[i];
    if(t.width <= 0 || t.height <= 0 || !t.rgba8)
      return refuse("texture without pixels");
    // the device keeps 16 levels (packTiled): a side of 65536 or more has a 17th, which would be sampled as level 15
    if(t.width >= 65536 || t.height >= 65536)
      return refuse("texture " + std::to_string(i) + " is " + std::to_string(t.width) + "x" + std::to_string(t.height)
                    + ": a side of 65536 or more needs more than the 16 mip levels the device stores");
    // the glTF sampler enums getSampler maps (src/gltf_scene_vk.cpp:922-945; anything else throws there)
    auto wrapOk = [](int m) { return m == 10497 || m == 33071 || m == 33648; };
    auto filterOk = [](int f) { return f == -1 || f == 9728 || f == 9729 || (f >= 9984 && f <= 9987); };
    if(!wrapOk(t.wrapS) || !wrapOk(t.wrapT) || !filterOk(t.magFilter) || !filterOk(t.minFilter))
      return refuse("texture " + std::to_string(i) + " has a sampler enum outside glTF's (wrap " + std::to_string(t.wrapS) + "/" + std::to_string(t.wrapT)
                    + ", filter " + std::to_string(t.magFilter) + "/" + std::to_string(t.minFilter) + ")");
  }
  for(uint32_t n = 0; n < s.numRenderNodes; n++)
  {
    if(s.renderNodeVisible && !s.renderNodeVisible[n])
      continue;
    const b200pt_render_node& node = s.renderNodes[n];
    if(node.renderPrimID < 0 || (uint32_t)node.renderPrimID >= s.numRenderPrimitives)
      return refuse("render node references a missing primitive");
    if(node.materialID >= (int)s.numMaterials)
      return refuse("render node references a missing material");
  }
  for(uint32_t i = 0; i < s.numRenderPrimitives; i++)
  {
    const b200pt_render_primitive& p = s.renderPrimitives[i];
    for(size_t k = 0; k < (size_t)p.triangleCount * 3; k++)
      if(p.indices[k] >= p.vertexCount)
        return refuse("b200pt_set_scene: index beyond the primitive's vertex count");
  }
  return validateMicromaps(h, "b200pt_set_scene", s);
}

// A path can take more than maxDepth wavefront iterations exactly when k_shade can scatter inside a medium: that is gated on the
// medium's scatter coefficient (multiscatterColorFactor) of a visible node's material, not on thickness (makeVolumeMedium runs on
// every transmission event, pathtrace_functions.h.slang:118-140, 605-672)
bool hasVolumeOf(const b200pt_scene_desc& s)
{
  for(uint32_t n = 0; n < s.numRenderNodes; n++)
  {
    if(s.renderNodeVisible && !s.renderNodeVisible[n])
      continue;
    const b200pt_shade_material& m = s.materials[materialOf(s.renderNodes[n])];
    if((m.transmissionFactor > 0.0f || m.transmissionTexture || m.diffuseTransmissionFactor > 0.0f || m.diffuseTransmissionTexture)
       && (m.multiscatterColorFactor[0] > 0.0f || m.multiscatterColorFactor[1] > 0.0f || m.multiscatterColorFactor[2] > 0.0f))
      return true;
  }
  return false;
}

// which KHR_materials_* features do the scene's materials use (reference: src/scene_feature_detection.cpp)
uint32_t featureMaskOf(const b200pt_scene_desc& s)
{
  uint32_t feat = s.numLights ? FEAT_LIGHTS : 0u;
  for(uint32_t i = 0; i < s.numMaterials; i++)
  {
    const b200pt_shade_material& m = s.materials[i];
    if(m.transmissionFactor > 0.0f || m.transmissionTexture)
      feat |= FEAT_TRANSMISSION;
    if(m.thicknessFactor > 0.0f || m.thicknessTexture || m.multiscatterColorFactor[0] > 0.0f || m.multiscatterColorFactor[1] > 0.0f || m.multiscatterColorFactor[2] > 0.0f)
      feat |= FEAT_VOLUME;
    if(m.diffuseTransmissionFactor > 0.0f || m.diffuseTransmissionTexture)
      feat |= FEAT_DIFFUSE_TRANSMISSION;
    if(m.clearcoatFactor > 0.0f)
      feat |= FEAT_CLEARCOAT;
    if(m.sheenColorFactor[0] != 0.0f || m.sheenColorFactor[1] != 0.0f || m.sheenColorFactor[2] != 0.0f)
      feat |= FEAT_SHEEN;
    if(m.iridescenceFactor > 0.0f)
      feat |= FEAT_IRIDESCENCE;
    if(m.anisotropyStrength > 0.0f)
      feat |= FEAT_ANISOTROPY;
    if(m.pbrModel == 1)
      feat |= FEAT_SPECGLOSS;
  }
  return feat;
}

// the feature variant of the shade kernel a frame runs: k_shade<0> when no material uses an extension feature, k_shade<FEAT_LEAN>
// when clearcoat is the only one, k_shade<FEAT_ALL> otherwise
static uint32_t shadeFeatures(const b200pt* h) { return h->featureMask == 0 ? 0u : h->leanShade ? (uint32_t)FEAT_LEAN : (uint32_t)FEAT_ALL; }

// the AoS tables (same bytes as the reference SSBOs) and the vertex data: separate attribute arrays per primitive, as
// SceneVk::createVertexBuffers
int uploadTables(b200pt* h, const b200pt_scene_desc& s, SceneBuild& b)
{
  DeviceArena&       A = b.mem;
  const cudaStream_t st = h->stream;
  b.nodesW = A.upload(s.renderNodes, s.numRenderNodes, st);
  b.S.nodes = b.nodesW;
  b.S.mats = b.tableMem.upload(s.materials, s.numMaterials, st);
  b.S.texInfos = b.tableMem.upload(s.textureInfos, s.numTextureInfos, st);
  b.S.lights = b.lightMem.upload(s.lights, s.numLights, st);
  b.S.numLights = (int)s.numLights;
  if(!b.tableMem.ok() || !b.lightMem.ok())
    return failed(h, b.tableMem.ok() ? b.lightMem : b.tableMem, "scene tables");
  b.primHost.resize(s.numRenderPrimitives);
  std::vector<DevPrim> prims(s.numRenderPrimitives);
  for(uint32_t i = 0; i < s.numRenderPrimitives; i++)
  {
    const b200pt_render_primitive& p = s.renderPrimitives[i];
    const size_t                   nv = p.vertexCount;
    DevPrim&                       d = prims[i];
    d.idx = A.upload(p.indices, (size_t)p.triangleCount * 3, st);
    d.pos = A.upload(p.positions, nv * 3, st);
    d.nrm = p.normals ? A.upload(p.normals, nv * 3, st) : nullptr;
    d.tan = p.tangents ? A.upload(p.tangents, nv * 4, st) : nullptr;
    d.uv0 = p.texCoords[0] ? A.upload(p.texCoords[0], nv * 2, st) : nullptr;
    d.uv1 = p.texCoords[1] ? A.upload(p.texCoords[1], nv * 2, st) : nullptr;
    d.col = p.colors ? A.upload(p.colors, nv, st) : nullptr;
    b.primHost[i].d = d;
    b.primHost[i].vertexCount = p.vertexCount;
    b.primHost[i].triCount = p.triangleCount;
  }
  b.S.prims = A.upload(prims.data(), prims.size(), st);
  return A.ok() ? B200PT_OK : failed(h, A, "scene tables and vertex arrays");
}

// mip chains and tiling on host threads, one allocation for all texels, one table of level offsets, the DevTex records
int uploadTextures(b200pt* h, const b200pt_scene_desc& s, SceneBuild& b)
{
  DeviceArena&             A = b.mem;
  std::vector<MipChain>    chains(s.numTextures);
  std::atomic<uint32_t>    nextTex{0};
  std::vector<std::thread> workers;
  auto                     job = [&]() {
    for(uint32_t i = nextTex.fetch_add(1); i < s.numTextures; i = nextTex.fetch_add(1))
      buildMipChain(s.textures[i], chains[i]);
  };
  const unsigned nt = std::max(1u, std::min(std::thread::hardware_concurrency(), s.numTextures));
  for(unsigned t = 1; t < nt; t++)
    workers.emplace_back(job);
  job();
  for(auto& t : workers)
    t.join();
  std::vector<uint32_t>              levelOfs((size_t)s.numTextures * 16, 0u);
  std::vector<size_t>                texBase(s.numTextures, 0);
  size_t                             total = 0;
  std::vector<std::vector<uint32_t>> packed(s.numTextures);
  {
    std::atomic<uint32_t>    nextPack{0};
    std::vector<std::thread> packers;
    auto                     pjob = [&]() {
      for(uint32_t i = nextPack.fetch_add(1); i < s.numTextures; i = nextPack.fetch_add(1))
        packTiled(chains[i], packed[i], &levelOfs[(size_t)i * 16]);
    };
    for(unsigned t = 1; t < nt; t++)
      packers.emplace_back(pjob);
    pjob();
    for(auto& t : packers)
      t.join();
  }
  for(uint32_t i = 0; i < s.numTextures; i++)
  {
    texBase[i] = total;
    total += packed[i].size();
  }
  uint32_t* dTexels = A.alloc<uint32_t>(total);
  if(!dTexels)
    return failed(h, A, "texels");
  for(uint32_t i = 0; i < s.numTextures; i++)
    CK(cudaMemcpy(dTexels + texBase[i], packed[i].data(), packed[i].size() * sizeof(uint32_t), cudaMemcpyHostToDevice));
  const uint32_t* dLevelOfs = A.upload(levelOfs.data(), levelOfs.size(), h->stream);
  if(!dLevelOfs)
    return failed(h, A, "texture level offsets");
  b.devTex.resize(s.numTextures);
  b.texLevel0.resize(s.numTextures);
  for(uint32_t i = 0; i < s.numTextures; i++)
  {
    describeTexture(s.textures[i], chains[i], b.devTex[i]);
    b.devTex[i].texels = reinterpret_cast<const uchar4*>(dTexels + texBase[i]);
    b.texLevel0[i] = b.devTex[i].texels + levelOfs[(size_t)i * 16];
    b.devTex[i].levelOfs = dLevelOfs + (size_t)i * 16;
  }
  b.S.textures = A.upload(b.devTex.data(), b.devTex.size(), h->stream);
  b.S.numTextures = (int)s.numTextures;
  return b.S.textures ? B200PT_OK : failed(h, A, "texture records");
}

// every visible render node's triangles in world space (TLAS/BLAS replacement): flatten order is the global triangle id
void flattenInstances(const b200pt_scene_desc& s, SceneBuild& b)
{
  for(uint32_t n = 0; n < s.numRenderNodes; n++)
  {
    if(s.renderNodeVisible && !s.renderNodeVisible[n])
      continue;
    const b200pt_render_node&      node = s.renderNodes[n];
    const b200pt_render_primitive& p = s.renderPrimitives[node.renderPrimID];
    const uint32_t                 flags = triFlags(s.materials[materialOf(node)]);
    const float*                   a = node.objectToWorld;
    const float  det = a[0] * (a[5] * a[10] - a[9] * a[6]) - a[4] * (a[1] * a[10] - a[9] * a[2]) + a[8] * (a[1] * a[6] - a[5] * a[2]);
    const bool   mirrored = det < 0.0f;
    for(uint32_t t = 0; t < p.triangleCount; t++)
    {
      float3 v[3];
      for(int k = 0; k < 3; k++)
      {
        const uint32_t vi = p.indices[t * 3 + k];
        v[k] = xfPoint(a, f3(p.positions[vi * 3], p.positions[vi * 3 + 1], p.positions[vi * 3 + 2]));
      }
      FlatTri T;
      T.rnode = n;
      T.prim = t;
      T.flags = flags;
      if(mirrored)
      {
        std::swap(v[1], v[2]);
        T.flags |= TRI_FLIPPED;
      }
      const float3 e1 = v[1] - v[0], e2 = v[2] - v[0];
      T.v0[0] = v[0].x, T.v0[1] = v[0].y, T.v0[2] = v[0].z;
      T.e1[0] = e1.x, T.e1[1] = e1.y, T.e1[2] = e1.z;
      T.e2[0] = e2.x, T.e2[1] = e2.y, T.e2[2] = e2.z;
      b.flat.push_back(T);
    }
  }
}

// ONE tree over every triangle (opaque and any-hit geometry alike: the per-triangle TRI_OPAQUE flag decides what a geometric hit
// means, traverse.cuh); the global triangle id (flatten order) is the tie-break key.  Closest-hit rays walk the merged tree;
// shadow rays walk an opaque-only tree first (any hit ends the query, occluded rays never meet the foliage boxes) and the
// non-opaque tree after it (traverse.cuh).  The three builds run in parallel.
int buildTrees(b200pt* h, SceneBuild& b)
{
  const std::vector<FlatTri>& flat = b.flat;
  std::vector<uint32_t>       gids(flat.size());
  for(uint32_t i = 0; i < (uint32_t)flat.size(); i++)
  {
    gids[i] = i;
    b.anyNonOpaque = b.anyNonOpaque || !(flat[i].flags & TRI_OPAQUE);
  }
  std::vector<FlatTri>  flatO, flatA;
  std::vector<uint32_t> gidO, gidA;
  if(b.anyNonOpaque)
    for(uint32_t i = 0; i < (uint32_t)flat.size(); i++)
    {
      if(flat[i].flags & TRI_OPAQUE)
      {
        flatO.push_back(flat[i]);
        gidO.push_back(i);
      }
      else
      {
        flatA.push_back(flat[i]);
        gidA.push_back(i);
      }
    }
  const auto tBuild0 = std::chrono::steady_clock::now();
  if(h->bvhBuilder == 1)
  {
    // device LBVH: the flattened records go up once (flatten order = global id order), the subsets as id lists
    std::vector<float> rec(flat.size() * 12);
    for(size_t i = 0; i < flat.size(); i++)
    {
      const FlatTri& T = flat[i];
      float*         R = &rec[i * 12];
      const uint32_t w0 = T.rnode | (T.flags << 28), prim = T.prim, gid = (uint32_t)i;
      memcpy(R, T.v0, 12);
      memcpy(R + 3, &w0, 4);
      memcpy(R + 4, T.e1, 12);
      memcpy(R + 7, &prim, 4);
      memcpy(R + 8, T.e2, 12);
      memcpy(R + 11, &gid, 4);
    }
    DeviceArena     tmp;
    const float*    dRec = tmp.upload(rec.data(), rec.size(), h->stream);
    const uint32_t* dO = b.anyNonOpaque ? tmp.upload(gidO.data(), gidO.size(), h->stream) : nullptr;
    const uint32_t* dA = b.anyNonOpaque ? tmp.upload(gidA.data(), gidA.size(), h->stream) : nullptr;
    int             rc = tmp.ok() ? B200PT_OK : failed(h, tmp, "GPU BVH build input");
    if(!rc)
      rc = buildWideBvhGpu(h, dRec, nullptr, (uint32_t)flat.size(), 0u, b.bvh);
    if(!rc && b.anyNonOpaque)
    {
      rc = buildWideBvhGpu(h, dRec, dO, (uint32_t)gidO.size(), 0u, b.bvhO);
      if(!rc)
        rc = buildWideBvhGpu(h, dRec, dA, (uint32_t)gidA.size(), (uint32_t)gidO.size(), b.bvhA);
    }
    cudaStreamSynchronize(h->stream);
    if(rc)
      return rc;
  }
  else
  {
    std::thread tO, tA;
    if(b.anyNonOpaque)
    {
      tO = std::thread([&] { buildWideBvh(flatO, gidO, 0u, b.bvhO); });
      tA = std::thread([&] { buildWideBvh(flatA, gidA, (uint32_t)flatO.size(), b.bvhA); });
    }
    buildWideBvh(flat, gids, 0u, b.bvh);
    if(b.anyNonOpaque)
    {
      tO.join();
      tA.join();
    }
  }
  b.bvhBuildMs = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tBuild0).count();
  return B200PT_OK;
}

// breadth-first level ranges of a tree (the builders emit level by level, so every level is one contiguous index range)
std::vector<std::pair<uint32_t, uint32_t>> levelsOf(const WideBvh& t)
{
  std::vector<std::pair<uint32_t, uint32_t>> lv;
  uint32_t                                   first = 0, count = 1;
  while(count)
  {
    lv.push_back({first, count});
    uint32_t next = 0;
    for(uint32_t n = first; n < first + count; n++)
    {
      uint32_t w;
      memcpy(&w, &t.nodes[(size_t)n * 20 + 3], 4);
      next += (uint32_t)__builtin_popcount(w >> 24);
    }
    first += count;
    count = next;
  }
  return lv;
}

// The node and triangle arrays of all three trees live in ONE allocation, so that a single L2 access-policy window can pin them
// (setTreeWindow): the walks re-read these few tens of MB all the time while every bounce streams GBs of path state past them.
// Also the trees' views for the refit (b200pt::TreeDev) with their level ranges and box scratch.
int packTrees(b200pt* h, SceneBuild& b)
{
  DeviceArena&       A = b.treeMem;
  const WideBvh &    bvh = b.bvh, &bvhO = b.bvhO, &bvhA = b.bvhA;
  std::vector<float> trisS, packed;
  size_t             offTris = 0, offNodesO = 0, offNodesA = 0, offTrisS = 0;
  auto               place = [&](const std::vector<float>& v) {
    const size_t at = packed.size();
    packed.insert(packed.end(), v.begin(), v.end());
    packed.resize((packed.size() + 31) & ~(size_t)31, 0.0f);  // 128-byte granules
    return at;
  };
  place(bvh.nodes);
  offTris = place(bvh.tris);
  std::vector<uint32_t> metaS;
  if(b.anyNonOpaque)
  {
    trisS = bvhO.tris;
    trisS.insert(trisS.end(), bvhA.tris.begin(), bvhA.tris.end());
    offNodesO = place(bvhO.nodes);
    offNodesA = place(bvhA.nodes);
    offTrisS = place(trisS);
    metaS = bvhO.triMeta;
    metaS.insert(metaS.end(), bvhA.triMeta.begin(), bvhA.triMeta.end());
  }
  float* const    dPacked = A.upload(packed.data(), packed.size(), h->stream);
  uint32_t* const dMeta = A.upload(bvh.triMeta.data(), bvh.triMeta.size(), h->stream);
  uint32_t* const dMetaS = b.anyNonOpaque ? A.upload(metaS.data(), metaS.size(), h->stream) : nullptr;
  if(!A.ok())
    return failed(h, A, "trees");
  b.treeBase = dPacked;
  b.treeBytes = packed.size() * sizeof(float);
  DevScene& S = b.S;
  S.bvh.nodes = reinterpret_cast<const float4*>(dPacked);
  S.bvh.tris = reinterpret_cast<const float4*>(dPacked + offTris);
  S.bvh.ommRef = nullptr;
  S.bvh.ommData = nullptr;
  S.bvh.capRef = nullptr;
  S.bvh.capBits = nullptr;
  S.hasAlpha = b.anyNonOpaque ? 1 : 0;
  S.triMeta = reinterpret_cast<const uint2*>(dMeta);
  S.bvhO = S.bvh;
  S.bvhA = S.bvh;
  S.triMetaS = S.triMeta;
  b.tree[0].nodes = dPacked;
  b.tree[0].tris = dPacked + offTris;
  b.tree[0].meta = reinterpret_cast<uint2*>(dMeta);
  b.tree[0].numNodes = bvh.numNodes;
  b.tree[0].numTriSlots = bvh.numTris;
  b.tree[0].levels = levelsOf(bvh);
  uint64_t splitNodeBytes = 0, splitTriBytes = 0;
  if(b.anyNonOpaque)
  {
    float *dNodesO = dPacked + offNodesO, *dNodesA = dPacked + offNodesA, *dTrisS = dPacked + offTrisS;
    S.bvhO.nodes = reinterpret_cast<const float4*>(dNodesO);
    S.bvhO.tris = reinterpret_cast<const float4*>(dTrisS);
    S.bvhA.nodes = reinterpret_cast<const float4*>(dNodesA);
    S.bvhA.tris = reinterpret_cast<const float4*>(dTrisS);
    S.triMetaS = reinterpret_cast<const uint2*>(dMetaS);
    splitNodeBytes = (bvhO.nodes.size() + bvhA.nodes.size()) * sizeof(float);
    splitTriBytes = trisS.size() * sizeof(float);
    b.tree[1].nodes = dNodesO;
    b.tree[1].tris = dTrisS;
    b.tree[1].meta = reinterpret_cast<uint2*>(dMetaS);
    b.tree[1].numNodes = bvhO.numNodes;
    b.tree[1].numTriSlots = bvhO.numTris + bvhA.numTris;  // the shared array is refitted once, through this entry
    b.tree[1].levels = levelsOf(bvhO);
    b.tree[2].nodes = dNodesA;
    b.tree[2].tris = dTrisS;
    b.tree[2].meta = nullptr;
    b.tree[2].numNodes = bvhA.numNodes;
    b.tree[2].numTriSlots = 0;
    b.tree[2].levels = levelsOf(bvhA);
  }
  for(auto& t : b.tree)
    if(t.nodes)
      t.nodeBox = A.alloc<float4>((size_t)std::max(t.numNodes, 1u) * 2);
  if(!A.ok())
    return failed(h, A, "refit boxes");
  b.nodeBytes = bvh.nodes.size() * sizeof(float) + splitNodeBytes;
  b.triBytes = bvh.tris.size() * sizeof(float) + splitTriBytes;
  return B200PT_OK;
}

// per-triangle attribute records for getHitState (device_scene.cuh: ShadeRec), per render primitive
int gatherShadeRecs(b200pt* h, const b200pt_scene_desc& s, SceneBuild& b)
{
  DeviceArena&          A = b.mem;
  std::vector<uint32_t> recBase(s.numRenderPrimitives, 0);
  size_t                total = 0;
  for(uint32_t i = 0; i < s.numRenderPrimitives; i++)
  {
    recBase[i] = (uint32_t)total;
    total += s.renderPrimitives[i].triangleCount;
  }
  std::vector<ShadeRec> recs(total);
  for(uint32_t i = 0; i < s.numRenderPrimitives; i++)
  {
    const b200pt_render_primitive& p = s.renderPrimitives[i];
    for(uint32_t t = 0; t < p.triangleCount; t++)
    {
      ShadeRec& r = recs[recBase[i] + t];
      float*    f = reinterpret_cast<float*>(&r);  // 48 floats, layout: device_scene.cuh ShadeRec
      memset(f, 0, sizeof(ShadeRec));
      const uint32_t flags = (p.normals ? 1u : 0u) | (p.texCoords[0] ? 2u : 0u) | (p.texCoords[1] ? 4u : 0u) | (p.colors ? 8u : 0u) | (p.tangents ? 16u : 0u);
      memcpy(&f[3], &flags, 4);
      uint32_t vi[3];
      for(int c = 0; c < 3; c++)
      {
        vi[c] = p.indices[t * 3 + c];
        memcpy(&f[c * 4], &p.positions[vi[c] * 3], 12);                 // v[0..2].xyz
        if(p.normals)
          memcpy(&f[12 + c * 4], &p.normals[vi[c] * 3], 12);            // v[3..5].xyz
        if(p.colors)
          memcpy(&f[7 + c * 4], &p.colors[vi[c]], 4);                   // v[1].w, v[2].w, v[3].w
        if(p.tangents)
          memcpy(&f[36 + c * 4], &p.tangents[vi[c] * 4], 16);           // v[9..11]
      }
      if(p.texCoords[0])
      {
        f[19] = p.texCoords[0][vi[0] * 2];                               // v[4].w
        f[23] = p.texCoords[0][vi[0] * 2 + 1];                           // v[5].w
        memcpy(&f[24], &p.texCoords[0][vi[1] * 2], 8);                   // v[6].xy
        memcpy(&f[26], &p.texCoords[0][vi[2] * 2], 8);                   // v[6].zw
      }
      if(p.texCoords[1])
      {
        memcpy(&f[28], &p.texCoords[1][vi[0] * 2], 8);                   // v[7].xy
        memcpy(&f[30], &p.texCoords[1][vi[1] * 2], 8);                   // v[7].zw
        memcpy(&f[32], &p.texCoords[1][vi[2] * 2], 8);                   // v[8].xy
      }
    }
  }
  b.shadeRecsW = A.upload(recs.data(), recs.size(), h->stream);
  b.S.shadeRecs = b.shadeRecsW;
  for(uint32_t i = 0; i < s.numRenderPrimitives; i++)
    b.primHost[i].recBase = recBase[i];
  return A.ok() ? B200PT_OK : failed(h, A, "shade records");
}

// the shade record and the material of every triangle slot of the merged tree
int gatherSlotRecs(b200pt* h, const b200pt_scene_desc& s, SceneBuild& b)
{
  DeviceArena&          A = b.treeMem;
  const WideBvh&        bvh = b.bvh;
  std::vector<uint32_t> idxOfSlot(bvh.numTris, 0u), matOfSlot(bvh.numTris, 0u);
  for(uint32_t k = 0; k < bvh.numTris; k++)
  {
    uint32_t gid;
    memcpy(&gid, &bvh.tris[(size_t)k * 12 + 11], 4);
    const b200pt_render_node& node = s.renderNodes[b.flat[gid].rnode];
    idxOfSlot[k] = b.primHost[node.renderPrimID].recBase + b.flat[gid].prim;
    matOfSlot[k] = materialOf(node);
  }
  b.S.shadeIdx = A.upload(idxOfSlot.data(), idxOfSlot.size(), h->stream);
  b.matOfSlotW = A.upload(matOfSlot.data(), matOfSlot.size(), h->stream);
  b.S.matOfSlot = b.matOfSlotW;
  b.S.numMaterials = (int)s.numMaterials;
  return A.ok() ? B200PT_OK : failed(h, A, "slot records");
}

// alpha-triangle records (device_scene.cuh: AlphaRec), one per non-opaque triangle in bvhA's leaf order
int gatherAlphaRecs(b200pt* h, const b200pt_scene_desc& s, SceneBuild& b)
{
  if(!b.anyNonOpaque)
    return B200PT_OK;
  DeviceArena&          A = b.treeMem;
  const WideBvh &       bvh = b.bvh, &bvhA = b.bvhA;
  const uint32_t        nA = bvhA.numTris;
  std::vector<AlphaRec> recs(nA);
  std::vector<uint32_t> recOfGid(b.flat.size(), 0xFFFFFFFFu);
  auto                  level0 = [&](int t) { return b.texLevel0[t]; };
  for(uint32_t k = 0; k < nA; k++)
  {
    uint32_t gid;
    memcpy(&gid, &bvhA.tris[(size_t)k * 12 + 11], 4);
    recOfGid[gid] = k;
    const FlatTri&                 T = b.flat[gid];
    const b200pt_render_node&      node = s.renderNodes[T.rnode];
    const b200pt_render_primitive& p = s.renderPrimitives[node.renderPrimID];
    recs[k] = alphaRecOf(s.materials[materialOf(node)], s.textureInfos, b.devTex.data(), s.numTextures, level0, p.texCoords[0], p.texCoords[1],
                         p.colors, p.indices[T.prim * 3], p.indices[T.prim * 3 + 1], p.indices[T.prim * 3 + 2]);
  }
  std::vector<uint32_t> idxOfSlot(bvh.numTris, 0xFFFFFFFFu);
  for(uint32_t k = 0; k < bvh.numTris; k++)
  {
    uint32_t gid;
    memcpy(&gid, &bvh.tris[(size_t)k * 12 + 11], 4);
    idxOfSlot[k] = recOfGid[gid];
  }
  b.alphaRecsW = A.upload(recs.data(), recs.size(), h->stream);
  b.S.alphaRecs = b.alphaRecsW;
  b.S.alphaIdx = A.upload(idxOfSlot.data(), idxOfSlot.size(), h->stream);
  b.S.alphaBaseS = b.bvhO.numTris;
  return A.ok() ? B200PT_OK : failed(h, A, "alpha records");
}

// opacity micromaps (omm.cuh): one reference word per triangle slot of the merged tree and of the shadow rays' arrays
int linkMicromaps(b200pt* h, const b200pt_scene_desc& s, SceneBuild& b)
{
  if(!b.anyNonOpaque || h->primOmms.empty())
    return B200PT_OK;
  DeviceArena&          A = b.treeMem;
  const WideBvh &       bvh = b.bvh, &bvhO = b.bvhO, &bvhA = b.bvhA;
  std::vector<uint8_t>  data;
  std::vector<uint32_t> dataBase(h->omms.size());
  for(size_t m = 0; m < h->omms.size(); m++)
  {
    dataBase[m] = (uint32_t)data.size();
    data.insert(data.end(), h->omms[m].data.begin(), h->omms[m].data.end());
  }
  data.resize(data.size() + 4, 0);  // (never read: keeps the allocation non-empty)
  std::vector<int> ommOfPrim(s.numRenderPrimitives, -1);
  for(size_t k = 0; k < h->primOmms.size(); k++)
    ommOfPrim[h->primOmms[k].prim] = (int)k;
  uint32_t linked = 0;
  auto     refOf = [&](uint32_t w0, uint32_t primTri) -> uint32_t {
    const uint32_t unknown = pt::kOmmNoLookup | (uint32_t)pt::OMM_UNKNOWN;
    if((w0 >> 28) & TRI_OPAQUE)
      return unknown;  // FORCE_OPAQUE instance: the walk never asks
    const int k = ommOfPrim[(uint32_t)s.renderNodes[w0 & 0x0fffffffu].renderPrimID];
    if(k < 0)
      return unknown;
    const auto&   po = h->primOmms[(size_t)k];
    const int32_t idx = po.hasIdx ? po.idx[primTri] : (int32_t)primTri;
    linked++;
    if(idx == B200PT_OMM_INDEX_FULLY_TRANSPARENT)
      return pt::kOmmNoLookup | (uint32_t)pt::OMM_TRANSPARENT;
    if(idx == B200PT_OMM_INDEX_FULLY_OPAQUE)
      return pt::kOmmNoLookup | (uint32_t)pt::OMM_OPAQUE;
    if(idx < 0)
      return unknown;
    const b200pt_micromap_triangle& T = h->omms[po.micromap].tris[(size_t)idx + po.base];
    return ((uint32_t)T.subdivisionLevel << 28) | (T.format == B200PT_OMM_FORMAT_4_STATE ? (1u << 27) : 0u) | (dataBase[po.micromap] + T.dataOffset);
  };
  std::vector<uint32_t> ref(bvh.numTris), refS((size_t)bvhO.numTris + bvhA.numTris, pt::kOmmNoLookup | (uint32_t)pt::OMM_UNKNOWN);
  for(uint32_t k = 0; k < bvh.numTris; k++)
    ref[k] = refOf(bvh.triMeta[(size_t)k * 2], bvh.triMeta[(size_t)k * 2 + 1]);
  b.ommTriangles = linked;
  for(uint32_t k = 0; k < bvhA.numTris; k++)
    refS[(size_t)bvhO.numTris + k] = refOf(bvhA.triMeta[(size_t)k * 2], bvhA.triMeta[(size_t)k * 2 + 1]);
  const uint8_t* dData = A.upload(data.data(), data.size(), h->stream);
  b.S.bvh.ommRef = A.upload(ref.data(), ref.size(), h->stream);
  b.S.bvh.ommData = dData;
  b.S.bvhA.ommRef = A.upload(refS.data(), refS.size(), h->stream);
  b.S.bvhA.ommData = dData;
  return A.ok() ? B200PT_OK : failed(h, A, "micromap references");
}

// the steps that build the trees and every per-slot table over them into b.treeMem, from the flattened visible triangles
int buildTreeArena(b200pt* h, const b200pt_scene_desc& s, SceneBuild& b)
{
  flattenInstances(s, b);
  int rc;
  if((rc = buildTrees(h, b)) || (rc = packTrees(h, b)) || (rc = gatherSlotRecs(h, s, b)) || (rc = gatherAlphaRecs(h, s, b)) || (rc = linkMicromaps(h, s, b)))
    return rc;
  CK(cudaStreamSynchronize(h->stream));
  return B200PT_OK;
}

// hands the tree arena of a build to the handle (after the last step that can fail); the previous one is freed
void commitTrees(b200pt* h, SceneBuild& b)
{
  h->treeMem = std::move(b.treeMem);
  DevScene& S = h->S;
  S.bvh = b.S.bvh;
  S.bvhO = b.S.bvhO;
  S.bvhA = b.S.bvhA;
  S.hasAlpha = b.S.hasAlpha;
  S.triMeta = b.S.triMeta;
  S.triMetaS = b.S.triMetaS;
  S.matOfSlot = b.S.matOfSlot;
  S.shadeIdx = b.S.shadeIdx;
  S.alphaRecs = b.S.alphaRecs;
  S.alphaIdx = b.S.alphaIdx;
  S.alphaBaseS = b.S.alphaBaseS;
  h->dAlphaRecsW = b.alphaRecsW;
  h->dMatOfSlotW = b.matOfSlotW;
  h->bvhBuildMs = b.bvhBuildMs;
  h->treeBase = b.treeBase;
  h->treeBytes = b.treeBytes;
  for(int t = 0; t < 3; t++)
    h->tree[t] = std::move(b.tree[t]);
  h->ommTriangles = b.ommTriangles;
  h->nodeBytes = b.nodeBytes;
  h->triBytes = b.triBytes;
  h->numNodes = b.bvh.numNodes + (b.anyNonOpaque ? b.bvhO.numNodes + b.bvhA.numNodes : 0u);
  h->numTris = b.bvh.numTris;
}

// what the materials, the lights and the node visibility decide outside the trees (commitScene and the scene edits)
void commitFeatures(b200pt* h, const b200pt_scene_desc& s)
{
  h->featureMask = featureMaskOf(s);
  h->leanShade = (h->featureMask & ~(uint32_t)FEAT_LEAN) == 0;
  h->hasVolume = hasVolumeOf(s);
}

// hands a built scene to the handle (after the last step that can fail)
void commitScene(b200pt* h, const b200pt_scene_desc& s, SceneBuild& b)
{
  h->sceneMem = std::move(b.mem);
  h->tableMem = std::move(b.tableMem);
  h->lightMem = std::move(b.lightMem);
  h->S = b.S;
  commitTrees(h, b);
  h->numTextureInfos = s.numTextureInfos;
  commitFeatures(h, s);
  h->primHost = std::move(b.primHost);
  h->devTex = std::move(b.devTex);
  h->texLevel0 = std::move(b.texLevel0);
  h->materials.assign(s.materials, s.materials + s.numMaterials);
  h->texInfos.assign(s.textureInfos, s.textureInfos + s.numTextureInfos);
  h->visible.assign(s.numRenderNodes, 1);
  if(s.renderNodeVisible)
    h->visible.assign(s.renderNodeVisible, s.renderNodeVisible + s.numRenderNodes);
  h->numSceneNodes = s.numRenderNodes;
  h->dNodesW = b.nodesW;
  h->dPrimsW = b.S.prims;
  h->dShadeRecsW = b.shadeRecsW;
  h->haveScene = true;
}

// Persisting-L2 window over the trees on every stream that runs walks (cudaAccessPolicyWindow: lines of the window are kept, the
// path-state traffic around them is what gets evicted).  hitRatio shrinks when the trees are larger than the carve-out.
void setTreeWindow(b200pt* h)
{
  if(!h->treeBytes)
    return;
  int maxPersist = 0, maxWindow = 0;
  cudaDeviceGetAttribute(&maxPersist, cudaDevAttrMaxPersistingL2CacheSize, h->device);
  cudaDeviceGetAttribute(&maxWindow, cudaDevAttrMaxAccessPolicyWindowSize, h->device);
  if(maxPersist > 0 && maxWindow > 0)
  {
    const size_t carve = std::min<size_t>((size_t)maxPersist, std::max<size_t>(h->treeBytes, (size_t)1 << 20));
    cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, carve);
    cudaStreamAttrValue attr{};
    attr.accessPolicyWindow.base_ptr = const_cast<void*>(h->treeBase);
    attr.accessPolicyWindow.num_bytes = std::min<size_t>(h->treeBytes, (size_t)maxWindow);
    attr.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)carve / (double)attr.accessPolicyWindow.num_bytes);
    attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
    attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
    cudaStreamSetAttribute(h->stream, cudaStreamAttributeAccessPolicyWindow, &attr);
    for(int l = 0; l < b200pt::kMaxLanes; l++)
      if(h->lanes[l].stream)
        cudaStreamSetAttribute(h->lanes[l].stream, cudaStreamAttributeAccessPolicyWindow, &attr);
    cudaGetLastError();  // (a refused window is not an error: the walks run without it)
  }
}

// The alpha caps and holes (alpha_caps.cuh) of the handle's scene, baked from its alpha records into h->capMem: the reference words of
// the closest-hit tree and of the shadow rays' triangle array, and the maps of the triangles whose micro-triangles are not all of one
// kind.  Called after every change of the alpha records (b200pt_set_scene, a scene edit that changed an alpha input, a rebuild): a
// stale map would skip texels that are no longer transparent or end walks at texels that are no longer opaque.  Scenes with opacity
// micromaps or without non-opaque triangles get none, and so does every scene while B200PT_ALPHA_CAPS=0 (caps and holes change no
// result: the switch lets the tests compare walks with and without them).  The records are baked kChunk at a time, so the unpacked
// maps in flight stay at kChunk x 256 B on the device and on the host whatever the scene's size.
// Returns an error code with h->err set on a failure; the handle is then left without caps.
int bakeAlphaCaps(b200pt* h)
{
  DevScene& S = h->S;
  for(BvhView* v : {&S.bvh, &S.bvhO, &S.bvhA})
    v->capRef = v->capBits = nullptr;
  h->capMem.release();
  const char* e = getenv("B200PT_ALPHA_CAPS");
  if(!S.hasAlpha || S.bvh.ommRef || !h->dAlphaRecsW || (e && atoi(e) == 0))
    return B200PT_OK;
  constexpr uint32_t kChunk = 1u << 16, kMapWords = 2 * kCapWords;
  const cudaStream_t st = h->stream;
  const uint32_t     nC = h->tree[0].numTriSlots, nS = h->tree[1].numTriSlots, base = S.alphaBaseS, nA = nS - base;
  if(nC >= kCandCapsSlots || nS >= kCandCapsSlots)
    return B200PT_OK;  // (the walks tag caps and holes in a candidate's slot bits)
  DeviceArena        scratch;
  uint32_t* const    dBits = scratch.alloc<uint32_t>((size_t)std::min(nA, kChunk) * kMapWords);
  uint8_t* const     dShadowOk = scratch.alloc<uint8_t>(std::min(nA, kChunk));
  if(!scratch.ok())
    return failed(h, scratch, "alpha caps");
  // per record and ray kind (closest-hit rays, shadow rays: no caps unless shadowOk): neither, all caps, all holes, or its map
  // appended to the packed maps
  std::vector<uint32_t> refOfRec(nA, kCapNone), refOfRecS(nA, kCapNone), packed, bits((size_t)std::min(nA, kChunk) * kMapWords);
  std::vector<uint8_t>  shadowOk(nA);
  bool                  any = false;
  auto                  refOf = [&](const uint32_t* m, bool capsToo) {
    uint32_t caps = 0, holes = 0;
    for(uint32_t w = 0; w < kCapWords; w++)
    {
      caps += capsToo ? (uint32_t)__builtin_popcount(m[w]) : 0u;
      holes += (uint32_t)__builtin_popcount(m[kCapWords + w]);
    }
    if(caps == 0 && holes == 0)
      return kCapNone;
    any = true;
    if(caps == kCapMicro || holes == kCapMicro)
      return caps ? kCapAll : kHoleAll;
    const uint32_t ref = (uint32_t)packed.size();
    packed.insert(packed.end(), m, m + kMapWords);
    if(!capsToo)
      std::fill(packed.begin() + ref, packed.begin() + ref + kCapWords, 0u);
    return ref;
  };
  for(uint32_t r0 = 0; r0 < nA; r0 += kChunk)
  {
    const uint32_t n = std::min(kChunk, nA - r0);
    CK(cudaMemsetAsync(dBits, 0, (size_t)n * kMapWords * sizeof(uint32_t), st));
    k_cap_bake<<<gridFor(h, 8), 256, 0, st>>>(S.alphaRecs + r0, n, dBits, dShadowOk);
    h->kernelLaunches++;
    CK(cudaGetLastError());
    CK(cudaMemcpyAsync(bits.data(), dBits, (size_t)n * kMapWords * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    CK(cudaMemcpyAsync(shadowOk.data() + r0, dShadowOk, n, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    for(uint32_t r = 0; r < n; r++)
    {
      const uint32_t* m = &bits[(size_t)r * kMapWords];
      refOfRec[r0 + r] = refOf(m, true);
      refOfRecS[r0 + r] = shadowOk[r0 + r] ? refOfRec[r0 + r] : refOf(m, false);
    }
  }
  if(!any)
    return B200PT_OK;
  std::vector<uint32_t> recOfSlot(nC), refC(nC, kCapNone), refS(nS, kCapNone);
  CK(cudaMemcpy(recOfSlot.data(), S.alphaIdx, nC * sizeof(uint32_t), cudaMemcpyDeviceToHost));
  for(uint32_t k = 0; k < nC; k++)
    if(recOfSlot[k] != 0xFFFFFFFFu)
      refC[k] = refOfRec[recOfSlot[k]];
  for(uint32_t r = 0; r < nA; r++)
    refS[base + r] = refOfRecS[r];
  DeviceArena     caps;
  const uint32_t* dRefC = caps.upload(refC.data(), refC.size(), st);
  const uint32_t* dRefS = caps.upload(refS.data(), refS.size(), st);
  const uint32_t* dPacked = caps.upload(packed.data(), packed.size(), st);
  if(!caps.ok())
    return failed(h, caps, "alpha caps");
  CK(cudaStreamSynchronize(st));  // (the uploads read the host vectors)
  h->capMem = std::move(caps);
  S.bvh.capRef = dRefC;
  S.bvh.capBits = dPacked;
  S.bvhA.capRef = dRefS;
  S.bvhA.capBits = dPacked;
  return B200PT_OK;
}

// The caps of a scene that has just been committed (b200pt_set_scene, a scene edit).  The scene is complete and renders exactly the same
// without them, so a failed bake (an allocation or a copy) does not undo or fail the call that committed it: the walks then run without
// caps until the next bake, and the failure stays readable in b200pt_last_error.
void commitAlphaCaps(b200pt* h)
{
  if(bakeAlphaCaps(h))
  {
    for(BvhView* v : {&h->S.bvh, &h->S.bvhO, &h->S.bvhA})
      v->capRef = v->capBits = nullptr;
    h->capMem.release();
    cudaGetLastError();
    h->err = "alpha caps not baked (the scene renders without them): " + h->err;
  }
}

}  // namespace
extern "C" {

int b200pt_set_scene(b200pt_t* h, const b200pt_scene_desc* s)
{
  if(!h || !s || s->numMaterials == 0 || (s->numRenderNodes && (!s->renderNodes || !s->renderPrimitives)))
  {
    if(h)
      h->err = "b200pt_set_scene: invalid scene description";
    return B200PT_E_INVALID;
  }
  if(const int rc = enter(h, true))
    return rc;
  freeScene(h);
  SceneBuild b;
  b.S = h->S;  // the environment and the sRGB table
  int rc;
  if((rc = validateScene(h, *s)) || (rc = uploadTables(h, *s, b)) || (rc = uploadTextures(h, *s, b)) || (rc = gatherShadeRecs(h, *s, b))
     || (rc = buildTreeArena(h, *s, b)))
    return rc;
  commitScene(h, *s, b);
  setTreeWindow(h);
  commitAlphaCaps(h);
  return B200PT_OK;
}

int b200pt_bvh_info(b200pt_t* h, uint64_t* node_bytes, uint64_t* tri_bytes, uint32_t* num_nodes, uint32_t* num_tris)
{
  if(!h || !h->haveScene)
    return B200PT_E_INVALID;
  if(node_bytes)
    *node_bytes = h->nodeBytes;
  if(tri_bytes)
    *tri_bytes = h->triBytes;
  if(num_nodes)
    *num_nodes = h->numNodes;
  if(num_tris)
    *num_tris = h->numTris;
  return B200PT_OK;
}

int b200pt_set_opacity_micromaps(b200pt_t* h, const b200pt_micromap* micromaps, uint32_t num_micromaps, const b200pt_primitive_omm* prims, uint32_t num_prims)
{
  if(!h || (num_micromaps && !micromaps) || (num_prims && !prims))
    return B200PT_E_INVALID;
  std::vector<b200pt_t::OmmHost>     omms(num_prims ? num_micromaps : 0u);
  std::vector<b200pt_t::PrimOmmHost> po(num_prims);
  uint64_t                           total = 0;
  for(size_t m = 0; m < omms.size(); m++)
  {
    const b200pt_micromap& M = micromaps[m];
    if((M.dataSize && !M.data) || (M.numTriangles && !M.triangles))
    {
      h->err = "b200pt_set_opacity_micromaps: micromap with a null array";
      return B200PT_E_INVALID;
    }
    for(uint32_t t = 0; t < M.numTriangles; t++)
    {
      const b200pt_micromap_triangle& T = M.triangles[t];
      if((T.format != B200PT_OMM_FORMAT_2_STATE && T.format != B200PT_OMM_FORMAT_4_STATE) || T.subdivisionLevel > B200PT_OMM_MAX_LEVEL)
      {
        h->err = "b200pt_set_opacity_micromaps: micromap triangle with an unknown format or a subdivision level above 12";
        return B200PT_E_INVALID;
      }
      const uint64_t bits = (1ull << (2 * T.subdivisionLevel)) * (T.format == B200PT_OMM_FORMAT_4_STATE ? 2u : 1u);
      if((uint64_t)T.dataOffset + (bits + 7) / 8 > M.dataSize)
      {
        h->err = "b200pt_set_opacity_micromaps: micromap triangle data beyond dataSize";
        return B200PT_E_INVALID;
      }
    }
    omms[m].data.assign(M.data, M.data + M.dataSize);
    omms[m].tris.assign(M.triangles, M.triangles + M.numTriangles);
    total += M.dataSize;
  }
  if(total >= (1ull << 27))
  {
    h->err = "b200pt_set_opacity_micromaps: more than 128 MiB of micromap data";
    return B200PT_E_UNSUPPORTED;
  }
  for(uint32_t i = 0; i < num_prims; i++)
  {
    const b200pt_primitive_omm& P = prims[i];
    if(P.micromap >= num_micromaps || (P.numIndices && !P.indices))
    {
      h->err = "b200pt_set_opacity_micromaps: primitive linkage references a micromap out of range";
      return B200PT_E_INVALID;
    }
    po[i].prim = P.renderPrimID;
    po[i].micromap = P.micromap;
    po[i].base = P.baseTriangle;
    po[i].hasIdx = P.indices != nullptr;
    if(P.indices)
      po[i].idx.assign(P.indices, P.indices + P.numIndices);
    for(int32_t v : po[i].idx)
      if(v < B200PT_OMM_INDEX_FULLY_UNKNOWN_OPAQUE || (v >= 0 && (uint64_t)v + P.baseTriangle >= micromaps[P.micromap].numTriangles))
      {
        h->err = "b200pt_set_opacity_micromaps: micromap index out of range";
        return B200PT_E_INVALID;
      }
  }
  h->omms.swap(omms);
  h->primOmms.swap(po);
  return B200PT_OK;
}

int b200pt_set_bvh_builder(b200pt_t* h, int kind)
{
  if(!h || (kind != 0 && kind != 1))
    return B200PT_E_INVALID;
  h->bvhBuilder = kind;
  return B200PT_OK;
}

int b200pt_bvh_build_ms(b200pt_t* h, double* ms)
{
  if(!h || !ms || !h->haveScene)
    return B200PT_E_INVALID;
  *ms = h->bvhBuildMs;
  return B200PT_OK;
}

// triangle records recomputed from the primitives' current vertices and the nodes' current transforms, then every tree
// refitted bottom-up (refit.cuh); synchronous
static int refitTrees(b200pt_t* h)
{
  cudaStream_t st = h->stream;
  for(int t = 0; t < 3; t++)
  {
    b200pt::TreeDev& T = h->tree[t];
    if(!T.nodes)
      continue;
    if(T.numTriSlots)
    {
      k_refit_tris<<<gridFor(h, 4), 256, 0, st>>>(T.tris, T.meta, T.numTriSlots, h->dNodesW, h->dPrimsW);
      h->kernelLaunches++;
    }
  }
  for(int t = 0; t < 3; t++)
  {
    b200pt::TreeDev& T = h->tree[t];
    if(!T.nodes)
      continue;
    for(size_t l = T.levels.size(); l-- > 0;)
    {
      const uint32_t count = T.levels[l].second;
      k_refit_level<<<(count + 127) / 128, 128, 0, st>>>(T.nodes, T.tris, T.nodeBox, T.levels[l].first, count);
      h->kernelLaunches++;
    }
  }
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));
  return B200PT_OK;
}

// the reference snapshots objectToWorld at the start of a frame whose transforms change (src/renderer.cpp:630-655): here the first
// transform update after a rendered frame copies the render nodes' current objectToWorld before it overwrites them, and the next
// frame reads the copy.  Runs on the handle's stream after syncAll, so no frame in flight still reads the previous copy.
static int snapshotPrevTransforms(b200pt_t* h)
{
  if(!h->renderedSinceUpdate || h->numSceneNodes == 0)
    return B200PT_OK;
  if(!h->dPrevO2W && !(h->dPrevO2W = h->sceneMem.alloc<float>((size_t)h->numSceneNodes * 16)))
    return failed(h, h->sceneMem, "previous transforms");
  k_snapshot_prev_transforms<<<(h->numSceneNodes + 255) / 256, 256, 0, h->stream>>>(h->dNodesW, h->dPrevO2W, h->numSceneNodes);
  h->kernelLaunches++;
  CK(cudaGetLastError());
  h->prevO2WValid = true;
  h->renderedSinceUpdate = false;
  return B200PT_OK;
}

int b200pt_update_transforms(b200pt_t* h, const b200pt_render_node* nodes, uint32_t num_nodes)
{
  if(!h || !h->haveScene || !nodes || num_nodes != h->numSceneNodes)
  {
    if(h)
      h->err = "b200pt_update_transforms: needs the scene's render-node count (materials / primitives of the nodes must not change)";
    return B200PT_E_INVALID;
  }
  if(const int rc = enter(h, true))
    return rc;
  cudaStream_t st = h->stream;
  if(const int rc = snapshotPrevTransforms(h))
    return rc;
  CK(cudaMemcpyAsync(h->dNodesW, nodes, (size_t)num_nodes * sizeof(b200pt_render_node), cudaMemcpyHostToDevice, st));
  return refitTrees(h);
}

int b200pt_set_node_hierarchy(b200pt_t* h, const b200pt_node_hierarchy* g)
{
  if(!h || !h->haveScene || !g || g->numNodes == 0 || g->numLevels == 0 || !g->parentIndices || !g->topoNodeOrder || !g->levelOffsets || !g->mappings)
  {
    if(h)
      h->err = "b200pt_set_node_hierarchy: needs a scene and a complete hierarchy description";
    return B200PT_E_INVALID;
  }
  if(const int rc = enter(h, true))
    return rc;
  h->graph = b200pt::Hierarchy{};
  auto fail = [&](const char* msg) {
    h->err = msg;
    return B200PT_E_INVALID;
  };
  // every node exactly once, parents in earlier levels, offsets monotone and complete
  if(g->levelOffsets[0] != 0 || g->levelOffsets[g->numLevels] != g->numNodes)
    return fail("b200pt_set_node_hierarchy: levelOffsets must run from 0 to numNodes");
  std::vector<int> levelOf(g->numNodes, -1);
  for(uint32_t l = 0; l < g->numLevels; l++)
  {
    if(g->levelOffsets[l + 1] < g->levelOffsets[l] || g->levelOffsets[l + 1] > g->numNodes)
      return fail("b200pt_set_node_hierarchy: levelOffsets must be monotone");
    for(uint32_t k = g->levelOffsets[l]; k < g->levelOffsets[l + 1]; k++)
    {
      const int n = g->topoNodeOrder[k];
      if(n < 0 || (uint32_t)n >= g->numNodes || levelOf[n] != -1)
        return fail("b200pt_set_node_hierarchy: topoNodeOrder must list every node once");
      levelOf[n] = (int)l;
    }
  }
  for(uint32_t n = 0; n < g->numNodes; n++)
  {
    const int p = g->parentIndices[n];
    if(p >= (int)g->numNodes || (p >= 0 && levelOf[p] >= levelOf[n]))
      return fail("b200pt_set_node_hierarchy: a parent must sit in an earlier level than its child");
  }
  for(uint32_t i = 0; i < h->numSceneNodes; i++)
  {
    const b200pt_render_node_mapping& m = g->mappings[i];
    if(m.nodeID < 0 || (uint32_t)m.nodeID >= g->numNodes || m.renderPrimID < 0 || (size_t)m.renderPrimID >= h->primHost.size() || m.materialID >= h->S.numMaterials)
      return fail("b200pt_set_node_hierarchy: render-node mapping out of range");
  }
  b200pt::Hierarchy  G;
  const cudaStream_t st = h->stream;
  G.dParents = G.mem.upload(g->parentIndices, g->numNodes, st);
  G.dTopo = G.mem.upload(g->topoNodeOrder, g->numNodes, st);
  static_assert(sizeof(RenderNodeMapping) == sizeof(b200pt_render_node_mapping), "mapping layout");
  G.dMappings = G.mem.upload(reinterpret_cast<const RenderNodeMapping*>(g->mappings), h->numSceneNodes, st);
  if(g->instLocalMatrices)
    G.dInstLocal = G.mem.upload(g->instLocalMatrices, (size_t)h->numSceneNodes * 16, st);
  G.dLocalMats = G.mem.alloc<float>((size_t)g->numNodes * 16);
  G.dWorldMats = G.mem.alloc<float>((size_t)g->numNodes * 16);
  if(!G.mem.ok())
    return failed(h, G.mem, "node hierarchy");
  G.levelOffsets.assign(g->levelOffsets, g->levelOffsets + g->numLevels + 1);
  G.numGraphNodes = g->numNodes;
  CK(cudaStreamSynchronize(st));
  h->graph = std::move(G);
  return B200PT_OK;
}

int b200pt_update_node_matrices(b200pt_t* h, const float* local_matrices)
{
  if(!h || !h->haveScene || h->graph.numGraphNodes == 0 || !local_matrices)
  {
    if(h)
      h->err = "b200pt_update_node_matrices: needs b200pt_set_node_hierarchy and the nodes' local matrices";
    return B200PT_E_INVALID;
  }
  if(const int rc = enter(h, true))
    return rc;
  cudaStream_t st = h->stream;
  if(const int rc = snapshotPrevTransforms(h))
    return rc;
  const b200pt::Hierarchy& G = h->graph;
  CK(cudaMemcpyAsync(G.dLocalMats, local_matrices, (size_t)G.numGraphNodes * 16 * sizeof(float), cudaMemcpyHostToDevice, st));
  for(size_t l = 0; l + 1 < G.levelOffsets.size(); l++)
  {
    const uint32_t count = G.levelOffsets[l + 1] - G.levelOffsets[l];
    if(!count)
      continue;
    k_propagate_level<<<(count + 255) / 256, 256, 0, st>>>(G.dLocalMats, G.dWorldMats, G.dParents, G.dTopo, G.levelOffsets[l], count);
    h->kernelLaunches++;
  }
  if(h->numSceneNodes)
  {
    k_update_render_nodes<<<(h->numSceneNodes + 255) / 256, 256, 0, st>>>(G.dWorldMats, G.dMappings, G.dInstLocal, h->dNodesW, h->numSceneNodes);
    h->kernelLaunches++;
  }
  CK(cudaGetLastError());
  return refitTrees(h);
}

}  // extern "C"
namespace {

// ---- scene edits (b200pt_update_materials, b200pt_update_node_materials, b200pt_set_node_visibility) -------------------------------
// An edited handle renders what a fresh b200pt_set_scene of the edited description renders.  Two paths:
//   in place  the visible set is unchanged and no visible triangle changes TRI_OPAQUE: the tables are replaced and k_retag_tris /
//             k_gather_alpha rewrite what the materials decide in the trees' triangle records and the alpha records;
//   rebuild   otherwise (shadow-tree membership, the alpha records and the micromap links follow TRI_OPAQUE): the tree arena is
//             built again by b200pt_set_scene's own steps, from the primitives' CURRENT vertices and the nodes' CURRENT transforms,
//             so an animated pose survives.  The per-primitive shade records are not touched (they may hold that pose).

// the scene the handle holds, as a scene description: the render nodes as the device has them (transforms and material ids may
// have moved since b200pt_set_scene), the host copies of the tables and the visibility; loadGeometry adds the primitives' current
// vertex data
struct CurrentScene
{
  std::vector<b200pt_render_node>      nodes;
  std::vector<b200pt_render_primitive> prims;
  std::vector<std::vector<uint32_t>>   idx, col;
  std::vector<std::vector<float>>      pos, uv0, uv1;
  b200pt_scene_desc                    desc{};
};

int loadCurrentScene(b200pt* h, CurrentScene& c)
{
  c.nodes.resize(h->numSceneNodes);
  CK(cudaMemcpy(c.nodes.data(), h->dNodesW, c.nodes.size() * sizeof(b200pt_render_node), cudaMemcpyDeviceToHost));
  c.prims.assign(h->primHost.size(), b200pt_render_primitive{});
  for(size_t i = 0; i < c.prims.size(); i++)
  {
    c.prims[i].triangleCount = h->primHost[i].triCount;
    c.prims[i].vertexCount = h->primHost[i].vertexCount;
  }
  b200pt_scene_desc& d = c.desc;
  d.renderNodes = c.nodes.data();
  d.numRenderNodes = h->numSceneNodes;
  d.renderNodeVisible = h->visible.data();
  d.renderPrimitives = c.prims.data();
  d.numRenderPrimitives = (uint32_t)c.prims.size();
  d.materials = h->materials.data();
  d.numMaterials = (uint32_t)h->materials.size();
  d.textureInfos = h->texInfos.data();
  d.numTextureInfos = (uint32_t)h->texInfos.size();
  d.numTextures = (uint32_t)h->S.numTextures;
  d.numLights = (uint32_t)h->S.numLights;
  return B200PT_OK;
}

// the vertex data a tree rebuild reads: indices, positions, texture coordinates and colours of every primitive
int loadGeometry(b200pt* h, CurrentScene& c)
{
  const size_t n = c.prims.size();
  c.idx.resize(n), c.col.resize(n), c.pos.resize(n), c.uv0.resize(n), c.uv1.resize(n);
  for(size_t i = 0; i < n; i++)
  {
    const b200pt::PrimHost& P = h->primHost[i];
    b200pt_render_primitive& p = c.prims[i];
    const size_t            nv = P.vertexCount;
    auto fetch = [&](auto& dst, const auto* src, size_t count) -> const typename std::decay_t<decltype(dst)>::value_type* {
      if(!src)
        return nullptr;
      dst.resize(count);
      return cudaMemcpy(dst.data(), src, count * sizeof(dst[0]), cudaMemcpyDeviceToHost) == cudaSuccess ? dst.data() : nullptr;
    };
    p.indices = fetch(c.idx[i], P.d.idx, (size_t)P.triCount * 3);
    p.positions = fetch(c.pos[i], P.d.pos, nv * 3);
    p.texCoords[0] = fetch(c.uv0[i], P.d.uv0, nv * 2);
    p.texCoords[1] = fetch(c.uv1[i], P.d.uv1, nv * 2);
    p.colors = fetch(c.col[i], P.d.col, nv);
    if(!p.indices || !p.positions || (P.d.uv0 && !p.texCoords[0]) || (P.d.uv1 && !p.texCoords[1]) || (P.d.col && !p.colors))
    {
      cudaGetLastError();
      h->err = "scene edit: reading the primitives' vertex data back failed";
      return B200PT_E_CUDA;
    }
  }
  return B200PT_OK;
}

// what the alpha record and the shadow cap reference of a triangle read from its material (alphaRecOf, the transmission test of
// bakeAlphaCaps) is the same for material ma of scene a and material mb of scene b
bool sameAlphaInputs(const b200pt_scene_desc& a, uint32_t ma, const b200pt_scene_desc& b, uint32_t mb)
{
  const b200pt_shade_material &x = a.materials[ma], &y = b.materials[mb];
  auto bits = [](float f) {
    uint32_t u;
    memcpy(&u, &f, 4);
    return u;
  };
  auto slot = [](const b200pt_shade_material& m) { return m.pbrModel == 1 ? m.pbrDiffuseTexture : m.pbrBaseColorTexture; };
  auto factor = [](const b200pt_shade_material& m) { return m.pbrModel == 1 ? m.pbrDiffuseFactor[3] : m.pbrBaseColorFactor[3]; };
  if(x.alphaMode != y.alphaMode || bits(x.alphaCutoff) != bits(y.alphaCutoff) || x.pbrModel != y.pbrModel || bits(factor(x)) != bits(factor(y))
     || bits(x.transmissionFactor) != bits(y.transmissionFactor) || slot(x) != slot(y))
    return false;
  const uint16_t s = slot(x);
  if(s == 0)
    return true;
  if(s >= a.numTextureInfos || s >= b.numTextureInfos)
    return s >= a.numTextureInfos && s >= b.numTextureInfos;
  return a.textureInfos[s].index == b.textureInfos[s].index && a.textureInfos[s].texCoord == b.textureInfos[s].texCoord;
}

// Applies an edit whose every argument has been checked: `next` is the current scene `cur` with the edit applied.  newTables:
// next's materials / texture infos replace the tables; newIds: the render nodes' material ids (`next`'s) are written to the device
// nodes and the hierarchy's mappings.  The replacements are built before anything is swapped, so a failed allocation leaves the
// scene as it was.
int applySceneEdit(b200pt* h, const char* who, CurrentScene& cur, const b200pt_scene_desc& next, bool newTables, const int32_t* newIds)
{
  const b200pt_scene_desc& old = cur.desc;
  bool                     rebuild = false;
  for(uint32_t n = 0; n < old.numRenderNodes && !rebuild; n++)
  {
    const bool v = next.renderNodeVisible[n] != 0;
    rebuild = v != (old.renderNodeVisible[n] != 0);
    if(v && !rebuild && old.renderPrimitives[next.renderNodes[n].renderPrimID].triangleCount)
      rebuild = ((triFlags(old.materials[materialOf(old.renderNodes[n])]) ^ triFlags(next.materials[materialOf(next.renderNodes[n])])) & TRI_OPAQUE) != 0;
  }
  if(rebuild)
    if(const int rc = validateMicromaps(h, who, next))
      return rc;
  // the alpha caps follow the alpha records: baked again after a rebuild, or when an in-place edit changed an alpha input of a visible node
  bool rebake = rebuild;
  for(uint32_t n = 0; n < old.numRenderNodes && !rebake; n++)
    if(next.renderNodeVisible[n] && old.renderPrimitives[next.renderNodes[n].renderPrimID].triangleCount)
      rebake = !sameAlphaInputs(old, materialOf(old.renderNodes[n]), next, materialOf(next.renderNodes[n]));
  const cudaStream_t st = h->stream;
  DeviceArena        tables;
  const b200pt_shade_material* dMats = h->S.mats;
  const b200pt_texture_info*   dTexInfos = h->S.texInfos;
  if(newTables)
  {
    dMats = tables.upload(next.materials, next.numMaterials, st);
    dTexInfos = tables.upload(next.textureInfos, next.numTextureInfos, st);
    if(!tables.ok())
      return failed(h, tables, who);
  }
  SceneBuild b;
  if(rebuild)
  {
    b.S = h->S;
    b.primHost = h->primHost;
    b.devTex = h->devTex;
    b.texLevel0 = h->texLevel0;
    int rc;
    if((rc = loadGeometry(h, cur)) || (rc = buildTreeArena(h, next, b)))
      return rc;
  }
  // nothing below allocates but the alpha-cap bake at the end, whose failure only leaves the committed scene without caps (commitAlphaCaps)
  if(newIds && next.numRenderNodes)
  {
    CK(cudaMemcpy2DAsync(reinterpret_cast<char*>(h->dNodesW) + offsetof(b200pt_render_node, materialID), sizeof(b200pt_render_node), newIds, sizeof(int32_t),
                         sizeof(int32_t), next.numRenderNodes, cudaMemcpyHostToDevice, st));
    // (or the next b200pt_update_node_matrices would write the old ids back)
    if(h->graph.dMappings)
      CK(cudaMemcpy2DAsync(reinterpret_cast<char*>(h->graph.dMappings) + offsetof(RenderNodeMapping, materialID), sizeof(RenderNodeMapping), newIds,
                           sizeof(int32_t), sizeof(int32_t), next.numRenderNodes, cudaMemcpyHostToDevice, st));
  }
  if(newTables)
  {
    h->tableMem = std::move(tables);
    h->S.mats = dMats;
    h->S.texInfos = dTexInfos;
    h->materials.assign(next.materials, next.materials + next.numMaterials);
    h->texInfos.assign(next.textureInfos, next.textureInfos + next.numTextureInfos);
    h->numTextureInfos = next.numTextureInfos;
  }
  h->visible.assign(next.renderNodeVisible, next.renderNodeVisible + next.numRenderNodes);
  commitFeatures(h, next);
  if(rebuild)
  {
    commitTrees(h, b);
    setTreeWindow(h);
  }
  else
  {
    const DevScene& S = h->S;
    for(int t = 0; t < 2; t++)
    {
      const b200pt::TreeDev& T = h->tree[t];
      if(T.nodes && T.numTriSlots)
      {
        k_retag_tris<<<gridFor(h, 4), 256, 0, st>>>(T.tris, T.meta, t == 0 ? h->dMatOfSlotW : nullptr, T.numTriSlots, h->dNodesW, S.mats);
        h->kernelLaunches++;
      }
    }
    if(h->dAlphaRecsW)
    {
      k_gather_alpha<<<gridFor(h, 4), 256, 0, st>>>(h->dAlphaRecsW, S.triMetaS, S.alphaBaseS, h->tree[1].numTriSlots - S.alphaBaseS, S);
      h->kernelLaunches++;
    }
  }
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(st));
  // (a stale map would make the walks skip what they must find; a rebuild's new arena starts without caps)
  if(rebake)
    commitAlphaCaps(h);
  return B200PT_OK;
}

}  // namespace
extern "C" {

int b200pt_update_materials(b200pt_t* h, const b200pt_shade_material* materials, uint32_t num_materials, const b200pt_texture_info* texture_infos,
                            uint32_t num_texture_infos)
{
  const char* who = "b200pt_update_materials";
  if(!h || !h->haveScene || !materials || num_materials != h->materials.size() || (num_texture_infos && !texture_infos))
  {
    if(h)
      h->err = std::string(who) + ": needs a scene and a material table of the scene's material count";
    return B200PT_E_INVALID;
  }
  int rc;
  if((rc = enter(h, true)) || (rc = validateMaterials(h, who, materials, num_materials, num_texture_infos)))
    return rc;
  CurrentScene cur;
  if((rc = loadCurrentScene(h, cur)))
    return rc;
  b200pt_scene_desc next = cur.desc;
  next.materials = materials;
  next.textureInfos = texture_infos;
  next.numTextureInfos = num_texture_infos;
  return applySceneEdit(h, who, cur, next, true, nullptr);
}

int b200pt_update_node_materials(b200pt_t* h, const int32_t* material_ids, uint32_t num_nodes)
{
  const char* who = "b200pt_update_node_materials";
  if(!h || !h->haveScene || (num_nodes && !material_ids) || num_nodes != h->numSceneNodes)
  {
    if(h)
      h->err = std::string(who) + ": needs a scene and one material id per render node";
    return B200PT_E_INVALID;
  }
  for(uint32_t n = 0; n < num_nodes; n++)
    if(material_ids[n] >= (int32_t)h->materials.size())
    {
      h->err = std::string(who) + ": render node references a missing material";
      return B200PT_E_INVALID;
    }
  int rc;
  CurrentScene cur;
  if((rc = enter(h, true)) || (rc = loadCurrentScene(h, cur)))
    return rc;
  std::vector<b200pt_render_node> nodes = cur.nodes;
  for(uint32_t n = 0; n < num_nodes; n++)
    nodes[n].materialID = material_ids[n];
  b200pt_scene_desc next = cur.desc;
  next.renderNodes = nodes.data();
  return applySceneEdit(h, who, cur, next, false, material_ids);
}

int b200pt_set_node_visibility(b200pt_t* h, const uint8_t* visible, uint32_t num_nodes)
{
  const char* who = "b200pt_set_node_visibility";
  if(!h || !h->haveScene || (num_nodes && !visible) || num_nodes != h->numSceneNodes)
  {
    if(h)
      h->err = std::string(who) + ": needs a scene and one flag per render node";
    return B200PT_E_INVALID;
  }
  int rc;
  CurrentScene cur;
  if((rc = enter(h, true)) || (rc = loadCurrentScene(h, cur)))
    return rc;
  std::vector<uint8_t> vis(num_nodes);
  for(uint32_t n = 0; n < num_nodes; n++)
  {
    vis[n] = visible[n] ? 1 : 0;
    // b200pt_set_scene checks visible nodes only: one that becomes visible is checked here
    const b200pt_render_node& node = cur.nodes[n];
    if(vis[n] && (node.renderPrimID < 0 || (uint32_t)node.renderPrimID >= cur.desc.numRenderPrimitives || node.materialID >= (int)cur.desc.numMaterials))
    {
      h->err = std::string(who) + ": a visible render node references a missing primitive or material";
      return B200PT_E_INVALID;
    }
  }
  b200pt_scene_desc next = cur.desc;
  next.renderNodeVisible = vis.data();
  return applySceneEdit(h, who, cur, next, false, nullptr);
}

int b200pt_update_lights(b200pt_t* h, const b200pt_light* lights, uint32_t num_lights)
{
  if(!h || !h->haveScene || (num_lights && !lights))
  {
    if(h)
      h->err = "b200pt_update_lights: needs a scene and the light array";
    return B200PT_E_INVALID;
  }
  if(const int rc = enter(h, true))
    return rc;
  DeviceArena         L;
  const b200pt_light* dLights = L.upload(lights, num_lights, h->stream);
  if(!L.ok())
    return failed(h, L, "b200pt_update_lights");
  CK(cudaStreamSynchronize(h->stream));
  h->lightMem = std::move(L);
  h->S.lights = dLights;
  h->S.numLights = (int)num_lights;
  h->featureMask = (h->featureMask & ~(uint32_t)FEAT_LIGHTS) | (num_lights ? (uint32_t)FEAT_LIGHTS : 0u);
  h->leanShade = (h->featureMask & ~(uint32_t)FEAT_LEAN) == 0;
  return B200PT_OK;
}

int b200pt_set_animation(b200pt_t* h, const b200pt_morph_task* morphs, uint32_t num_morphs, const b200pt_skin_task* skins, uint32_t num_skins)
{
  if(!h || !h->haveScene || (num_morphs && !morphs) || (num_skins && !skins))
  {
    if(h)
      h->err = "b200pt_set_animation: needs a scene (b200pt_set_scene first) and task arrays";
    return B200PT_E_INVALID;
  }
  if(const int rc = enter(h, true))
    return rc;
  h->anim = b200pt::Animation{};
  auto fail = [&](const char* msg) {
    h->err = msg;
    return B200PT_E_INVALID;
  };
  b200pt::Animation  a;
  DeviceArena&       A = a.mem;
  const cudaStream_t st = h->stream;
  for(uint32_t i = 0; i < num_morphs; i++)
  {
    const b200pt_morph_task& m = morphs[i];
    if(m.renderPrimID >= h->primHost.size())
      return fail("b200pt_set_animation: morph task for a render primitive out of range");
    const b200pt::PrimHost& P = h->primHost[m.renderPrimID];
    if(m.vertexCount != P.vertexCount || !m.basePositions || (m.numTargets && !m.positionDeltas))
      return fail("b200pt_set_animation: morph task needs base positions, position deltas and the primitive's vertex count");
    MorphTaskDev T{};
    T.vertexCount = m.vertexCount;
    T.numTargets = m.numTargets;
    const size_t nv = m.vertexCount, nd = (size_t)m.numTargets * m.vertexCount * 3;
    T.basePos = A.upload(m.basePositions, nv * 3, st);
    if(m.baseNormals && P.d.nrm)
      T.baseNrm = A.upload(m.baseNormals, nv * 3, st);
    if(m.baseTangents && P.d.tan)
      T.baseTan = A.upload(m.baseTangents, nv * 4, st);
    T.dPos = A.upload(m.positionDeltas, nd, st);
    if(m.normalDeltas && T.baseNrm)
      T.dNrm = A.upload(m.normalDeltas, nd, st);
    if(m.tangentDeltas && T.baseTan)
      T.dTan = A.upload(m.tangentDeltas, nd, st);
    T.outPos = const_cast<float*>(P.d.pos);
    T.outNrm = const_cast<float*>(P.d.nrm);
    T.outTan = const_cast<float*>(P.d.tan);
    a.numMorphWeights += m.numTargets;
    a.morphTasks.push_back(T);
    a.morphPrim.push_back(m.renderPrimID);
  }
  for(uint32_t i = 0; i < num_skins; i++)
  {
    const b200pt_skin_task& k = skins[i];
    if(k.renderPrimID >= h->primHost.size())
      return fail("b200pt_set_animation: skin task for a render primitive out of range");
    const b200pt::PrimHost& P = h->primHost[k.renderPrimID];
    if(k.vertexCount != P.vertexCount || !k.basePositions || !k.weights || !k.joints || k.numJoints == 0)
      return fail("b200pt_set_animation: skin task needs base positions, weights, joints and the primitive's vertex count");
    SkinTaskDev  T{};
    const size_t nv = k.vertexCount;
    T.vertexCount = k.vertexCount;
    T.numJoints = k.numJoints;
    T.basePos = A.upload(k.basePositions, nv * 3, st);
    if(k.baseNormals && P.d.nrm)
      T.baseNrm = A.upload(k.baseNormals, nv * 3, st);
    if(k.baseTangents && P.d.tan)
      T.baseTan = A.upload(k.baseTangents, nv * 4, st);
    T.weights = A.upload(k.weights, nv * 4, st);
    T.joints = A.upload(k.joints, nv * 4, st);
    T.outPos = const_cast<float*>(P.d.pos);
    T.outNrm = const_cast<float*>(P.d.nrm);
    T.outTan = const_cast<float*>(P.d.tan);
    a.numJoints += k.numJoints;
    a.skinTasks.push_back(T);
    a.skinPrim.push_back(k.renderPrimID);
  }
  // the per-frame buffers, sized once (createAnimationResources: totalJointMatBytes / totalNormalMatBytes / morph weights)
  a.dMorphWeights = A.alloc<float>(a.numMorphWeights);
  a.dJointMats = A.alloc<float>(a.numJoints * 16);
  a.dNormalMats = A.alloc<float>(a.numJoints * 9);
  if(!A.ok())
    return failed(h, A, "animation");
  size_t wOfs = 0, jOfs = 0;
  for(auto& T : a.morphTasks)
  {
    T.weights = a.dMorphWeights + wOfs;
    wOfs += T.numTargets;
  }
  for(auto& T : a.skinTasks)
  {
    T.jointMatrices = a.dJointMats + jOfs * 16;
    T.normalMatrices = a.dNormalMats + jOfs * 9;
    jOfs += T.numJoints;
  }
  CK(cudaStreamSynchronize(st));
  h->anim = std::move(a);
  return B200PT_OK;
}

int b200pt_animate(b200pt_t* h, const float* morph_weights, const float* joint_matrices, const float* normal_matrices)
{
  if(!h || !h->haveScene || (h->anim.morphTasks.empty() && h->anim.skinTasks.empty()) || (h->anim.numMorphWeights && !morph_weights)
     || (h->anim.numJoints && (!joint_matrices || !normal_matrices)))
  {
    if(h)
      h->err = "b200pt_animate: needs b200pt_set_animation and the per-frame weights / joint matrices / normal matrices of its tasks";
    return B200PT_E_INVALID;
  }
  if(const int rc = enter(h, true))
    return rc;
  const b200pt::Animation& a = h->anim;
  cudaStream_t             st = h->stream;
  // Phase 1 (gltf_scene_animation_vk.cpp:430-494): one upload of all per-frame data
  if(a.numMorphWeights)
    CK(cudaMemcpyAsync(a.dMorphWeights, morph_weights, a.numMorphWeights * sizeof(float), cudaMemcpyHostToDevice, st));
  if(a.numJoints)
  {
    CK(cudaMemcpyAsync(a.dJointMats, joint_matrices, a.numJoints * 16 * sizeof(float), cudaMemcpyHostToDevice, st));
    CK(cudaMemcpyAsync(a.dNormalMats, normal_matrices, a.numJoints * 9 * sizeof(float), cudaMemcpyHostToDevice, st));
  }
  // Phase 2 (:497-533): morph
  std::vector<uint8_t> touched(h->primHost.size(), 0), morphed(h->primHost.size(), 0);
  for(size_t i = 0; i < a.morphTasks.size(); i++)
  {
    const MorphTaskDev& T = a.morphTasks[i];
    if(T.numTargets == 0)
      continue;  // (:508) nothing to blend: the vertex buffers keep what they hold
    k_morph<<<(T.vertexCount + 255) / 256, 256, 0, st>>>(T);
    h->kernelLaunches++;
    touched[a.morphPrim[i]] = morphed[a.morphPrim[i]] = 1;
  }
  // Phase 3 (:536-582): skin; a primitive morphed above is skinned from its own (morphed) arrays
  for(size_t i = 0; i < a.skinTasks.size(); i++)
  {
    SkinTaskDev T = a.skinTasks[i];
    if(morphed[a.skinPrim[i]])
    {
      const DevPrim& P = h->primHost[a.skinPrim[i]].d;
      T.basePos = P.pos;
      T.baseNrm = P.nrm ? P.nrm : T.baseNrm;
      T.baseTan = P.tan ? P.tan : T.baseTan;
    }
    k_skin<<<(T.vertexCount + 255) / 256, 256, 0, st>>>(T);
    h->kernelLaunches++;
    touched[a.skinPrim[i]] = 1;
  }
  // the per-triangle shade records of the touched primitives follow their vertex arrays
  for(size_t p = 0; p < touched.size(); p++)
    if(touched[p] && h->primHost[p].triCount)
    {
      const b200pt::PrimHost& P = h->primHost[p];
      k_regather_shade<<<(P.triCount + 255) / 256, 256, 0, st>>>(h->dShadeRecsW + P.recBase, P.d, P.triCount);
      h->kernelLaunches++;
    }
  CK(cudaGetLastError());
  // the BLAS update the reference records after the compute barrier (:586-590): triangle records + bottom-up refit
  return refitTrees(h);
}

int b200pt_set_environment(b200pt_t* h, const float* rgb, int w, int hh, float* integral_out)
{
  if(!h || !rgb || w <= 0 || hh <= 0)
    return B200PT_E_INVALID;
  if(const int rc = enter(h, true))
    return rc;
  const size_t n = (size_t)w * hh;
  // importance = texel solid angle * max(r,g,b); Vose alias table; pdf stored in alpha
  // (nvvk::HdrIbl, external to the reference tree; call site src/renderer.cpp:1994-1996)
  std::vector<float>  rgba(n * 4), importance(n), q(n);
  std::vector<uint32_t> alias(n);
  const float         stepPhi = kTwoPi / (float)w, stepTheta = kPi / (float)hh;
  for(int y = 0; y < hh; y++)
  {
    const float theta0 = (float)y * stepTheta, theta1 = (float)(y + 1) * stepTheta;
    const float area = (cosf(theta0) - cosf(theta1)) * stepPhi;
    for(int x = 0; x < w; x++)
    {
      const size_t i = (size_t)y * w + x;
      const float  r = rgb[i * 3], g = rgb[i * 3 + 1], b = rgb[i * 3 + 2];
      rgba[i * 4] = r;
      rgba[i * 4 + 1] = g;
      rgba[i * 4 + 2] = b;
      importance[i] = area * std::max(r, std::max(g, b));
    }
  }
  float sum = 0.f;
  for(float d : importance)
    sum += d;
  const float average = sum / (float)n;
  for(size_t i = 0; i < n; i++)
  {
    q[i] = importance[i] / average;
    alias[i] = (uint32_t)i;
  }
  {
    std::vector<uint32_t> part(n);
    uint32_t              s = 0u, large = (uint32_t)n;
    for(uint32_t i = 0; i < (uint32_t)n; ++i)
    {
      if(q[i] < 1.f)
        part[s++] = i;
      else
        part[--large] = i;
    }
    for(s = 0; s < large && large < (uint32_t)n; ++s)
    {
      const uint32_t j = part[s], k = part[large];
      alias[j] = k;
      const float diff = 1.f - q[j];
      q[k] -= diff;
      if(q[k] < 1.0f)
        large++;
    }
  }
  const float inv = 1.0f / sum;
  for(size_t i = 0; i < n; i++)
    rgba[i * 4 + 3] = std::max(rgba[i * 4], std::max(rgba[i * 4 + 1], rgba[i * 4 + 2])) * inv;
  std::vector<uint32_t> accel(n * 2);
  for(size_t i = 0; i < n; i++)
  {
    accel[i * 2] = alias[i];
    memcpy(&accel[i * 2 + 1], &q[i], 4);
  }
  // the old environment goes first (peak memory stays one environment); until the new one is complete there is none
  h->envMem.release();
  h->haveEnv = false;
  h->S.envRgba = nullptr;
  h->S.envAccel = nullptr;
  DeviceArena   A;
  float4* const dEnv = A.alloc<float4>(n);
  uint2* const  dEnvAccel = A.alloc<uint2>(n);
  if(!A.ok())
    return failed(h, A, "environment");
  CK(cudaMemcpy(dEnv, rgba.data(), n * sizeof(float4), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dEnvAccel, accel.data(), n * sizeof(uint2), cudaMemcpyHostToDevice));
  h->envMem = std::move(A);
  h->S.envRgba = dEnv;
  h->S.envAccel = dEnvAccel;
  h->S.envW = w;
  h->S.envH = hh;
  h->haveEnv = true;
  if(integral_out)
    *integral_out = sum;
  return B200PT_OK;
}

int b200pt_resize(b200pt_t* h, int width, int height, int tile_y0, int tile_rows)
{
  if(!h || width <= 0 || height <= 0 || tile_y0 < 0 || tile_rows <= 0 || tile_y0 + tile_rows > height)
  {
    if(h)
      h->err = "b200pt_resize: invalid extent / tile";
    return B200PT_E_INVALID;
  }
  if(const int rc = enter(h, true))
    return rc;
  freePool(h);
  const size_t n = (size_t)width * tile_rows;          // pixels of the tile: image-sized buffers
  const size_t nPool = n * (size_t)std::max(h->batch, h->views);  // path slots per lane (at most one of the two is above 1)
  // nothing of the handle's geometry is committed before every allocation has succeeded: a failed resize leaves
  // numPaths == 0 and null pointers, so later calls fail their guards instead of touching freed memory
  DeviceArena A;
  PathState   P[b200pt::kMaxLanes];
  uint32_t*   dQ[b200pt::kMaxLanes][6] = {};
  ViewPose*   poses[b200pt::kMaxLanes] = {};
  for(int l = 0; l < h->numLanes; l++)
  {
    allocPathState(h, A, nPool, P[l]);
    for(int k = 0; k < 6; k++)
      dQ[l][k] = A.alloc<uint32_t>(nPool);
    if(h->views > 1)
      poses[l] = A.alloc<ViewPose>((size_t)h->views);
  }
  if(!A.ok())
    return failed(h, A, "path pool");
  float4* const accum = A.alloc<float4>(n);
  if(!accum)
    return failed(h, A, "accumulation image");
  uint32_t* const select = A.alloc<uint32_t>(n);
  if(!select)
    return failed(h, A, "selection image");
  float* const ndcDepth = A.alloc<float>(n);
  if(!ndcDepth)
    return failed(h, A, "depth image");
  float4* const  guide = h->guides ? A.alloc<float4>(n) : nullptr;
  if(h->guides && !guide)
    return failed(h, A, "guide image");
  const size_t   dlssBytes = n * kDlssBytesPerPixel + 6 * 256;
  uint8_t* const dlss = h->dlss ? A.alloc<uint8_t>(dlssBytes) : nullptr;
  if(h->dlss && !dlss)
    return failed(h, A, "DLSS guide images");
  uchar4* const tonemapped = A.alloc<uchar4>(n);
  if(!tonemapped)
    return failed(h, A, "tonemapped image");
  const size_t    nv = n * (size_t)(h->views - 1);  // pixels of views 1..
  float4* const   viewAccum = nv ? A.alloc<float4>(nv) : nullptr;
  uint32_t* const viewSelect = nv ? A.alloc<uint32_t>(nv) : nullptr;
  float* const    viewDepth = nv ? A.alloc<float>(nv) : nullptr;
  if(nv && !A.ok())
    return failed(h, A, "view images");
  const cudaStream_t st = h->stream;
  if((guide && cudaMemsetAsync(guide, 0, n * 16, st) != cudaSuccess) || (dlss && cudaMemsetAsync(dlss, 0, dlssBytes, st) != cudaSuccess)
     || cudaMemsetAsync(select, 0, n * 4, st) != cudaSuccess || cudaMemsetAsync(ndcDepth, 0, n * 4, st) != cudaSuccess
     || cudaMemsetAsync(accum, 0, n * 16, st) != cudaSuccess
     || (nv && (cudaMemsetAsync(viewAccum, 0, nv * 16, st) != cudaSuccess || cudaMemsetAsync(viewSelect, 0, nv * 4, st) != cudaSuccess
                || cudaMemsetAsync(viewDepth, 0, nv * 4, st) != cudaSuccess))
     || cudaStreamSynchronize(st) != cudaSuccess)
  {
    h->err = "b200pt_resize: clearing the new images failed";
    return B200PT_E_CUDA;
  }
  h->poolMem = std::move(A);
  for(int l = 0; l < h->numLanes; l++)
  {
    h->lanes[l].P = P[l];
    std::copy(dQ[l], dQ[l] + 6, h->lanes[l].dQ);
    h->lanes[l].poses = poses[l];
  }
  h->dViewAccum = viewAccum;
  h->dViewSelect = viewSelect;
  h->dViewDepth = viewDepth;
  h->dAccumOwned = accum;
  h->dSelect = select;
  h->dNdcDepth = ndcDepth;
  h->dGuide = guide;
  h->dDlss = dlss;
  h->dTonemapped = tonemapped;
  h->width = width;
  h->height = height;
  h->tileY0 = tile_y0;
  h->tileRows = tile_rows;
  h->bandRows = 0;
  h->bandWorld = 1;
  h->bandRank = 0;
  h->numPaths = (uint32_t)n;
  h->dAccum = h->dAccumOwned;
  return B200PT_OK;
}

int b200pt_resize_interleaved(b200pt_t* h, int width, int height, int band_rows, int world, int rank)
{
  if(!h || width <= 0 || height <= 0 || band_rows <= 0 || world <= 0 || rank < 0 || rank >= world || height % (band_rows * world) != 0)
  {
    if(h)
      h->err = "b200pt_resize_interleaved: height must be a multiple of band_rows * world, 0 <= rank < world";
    return B200PT_E_INVALID;
  }
  const int rc = b200pt_resize(h, width, height, 0, height / world);
  if(rc)
    return rc;
  h->bandRows = band_rows;
  h->bandWorld = world;
  h->bandRank = rank;
  return B200PT_OK;
}

int b200pt_set_accum_device(b200pt_t* h, float* dev, size_t num_floats)
{
  if(!h || h->numPaths == 0)
    return B200PT_E_INVALID;
  if(dev == nullptr)
  {
    h->dAccum = h->dAccumOwned;
    return B200PT_OK;
  }
  if(const int rc = enter(h, false))
    return rc;
  if(num_floats < (size_t)h->numPaths * 4)
  {
    h->err = "b200pt_set_accum_device: buffer too small";
    return B200PT_E_INVALID;
  }
  h->dAccum = reinterpret_cast<float4*>(dev);
  return B200PT_OK;
}

int b200pt_get_accum_device(b200pt_t* h, float** dev, size_t* num_floats)
{
  if(!h || h->numPaths == 0)
    return B200PT_E_INVALID;
  if(dev)
    *dev = reinterpret_cast<float*>(h->dAccum);
  if(num_floats)
    *num_floats = (size_t)h->numPaths * 4;
  return B200PT_OK;
}

int b200pt_read_accum(b200pt_t* h, float* host, size_t num_floats)
{
  if(!h || h->numPaths == 0 || !host || num_floats < (size_t)h->numPaths * 4)
    return B200PT_E_INVALID;
  if(const int rc = enter(h, false))
    return rc;
  CK(cudaMemcpyAsync(host, h->dAccum, (size_t)h->numPaths * 16, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return B200PT_OK;
}

// histogram (when auto-exposure is on) -> exposure factor -> operator + UNORM8 store, on the handle's stream
static int tonemapOnDevice(b200pt_t* h, const b200pt_tonemapper* tm, const float4* img, int width, int rows, int y0, int fullHeight, uchar4* out, float* exposure_used)
{
  if(tm->method < 0 || tm->method > 5 || !(tm->brightness > 0.0f))
  {
    h->err = "b200pt_tonemap: method must be 0..5 and brightness > 0";
    return B200PT_E_INVALID;
  }
  cudaStream_t   st = h->stream;
  const uint32_t n = (uint32_t)width * (uint32_t)rows;
  float*         dExposure = reinterpret_cast<float*>(h->dTmHist + kTmBins);
  if(tm->autoExposure && tm->isActive)
  {
    CK(cudaMemsetAsync(h->dTmHist, 0, kTmBins * sizeof(uint32_t), st));
    k_tm_histogram<<<gridFor(h, 8), 256, 0, st>>>(img, n, h->dTmHist);
    k_tm_exposure<<<1, 32, 0, st>>>(h->dTmHist, tm->exposure, dExposure);
    h->kernelLaunches += 2;
  }
  else
    CK(cudaMemcpyAsync(dExposure, &tm->exposure, sizeof(float), cudaMemcpyHostToDevice, st));
  k_tonemap<<<gridFor(h, 8), 256, 0, st>>>(img, out, width, rows, y0, fullHeight, *tm, dExposure);
  h->kernelLaunches++;
  CK(cudaGetLastError());
  if(exposure_used)
    CK(cudaMemcpyAsync(exposure_used, dExposure, sizeof(float), cudaMemcpyDeviceToHost, st));
  CK(cudaStreamSynchronize(st));
  return B200PT_OK;
}

int b200pt_tonemap(b200pt_t* h, const b200pt_tonemapper* tm, uint8_t* host_rgba8, size_t num_bytes, float* exposure_used)
{
  if(!h || !tm || h->numPaths == 0 || (host_rgba8 && num_bytes < (size_t)h->numPaths * 4))
    return B200PT_E_INVALID;
  if(h->bandWorld > 1)
  {
    h->err = "b200pt_tonemap: an interleaved multi-GPU tile is tonemapped after the gather (b200pt_tonemap_image on the full image)";
    return B200PT_E_UNSUPPORTED;
  }
  if(const int rc = enter(h, false))
    return rc;
  const int rc = tonemapOnDevice(h, tm, h->dAccum, h->width, h->tileRows, h->tileY0, h->height, h->dTonemapped, exposure_used);
  if(rc)
    return rc;
  if(host_rgba8)
  {
    CK(cudaMemcpyAsync(host_rgba8, h->dTonemapped, (size_t)h->numPaths * 4, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
  }
  return B200PT_OK;
}

int b200pt_tonemap_image(b200pt_t* h, const b200pt_tonemapper* tm, const float* dev_rgba32f, int width, int height, uint8_t* dev_rgba8, float* exposure_used)
{
  if(!h || !tm || !dev_rgba32f || !dev_rgba8 || width <= 0 || height <= 0)
    return B200PT_E_INVALID;
  CK(cudaSetDevice(h->device));
  return tonemapOnDevice(h, tm, reinterpret_cast<const float4*>(dev_rgba32f), width, height, 0, height, reinterpret_cast<uchar4*>(dev_rgba8), exposure_used);
}

int b200pt_get_tonemapped_device(b200pt_t* h, uint8_t** dev_rgba8, size_t* num_bytes)
{
  if(!h || h->numPaths == 0 || !dev_rgba8)
    return B200PT_E_INVALID;
  *dev_rgba8 = reinterpret_cast<uint8_t*>(h->dTonemapped);
  if(num_bytes)
    *num_bytes = (size_t)h->numPaths * 4;
  return B200PT_OK;
}

int b200pt_read_selection(b200pt_t* h, uint32_t* host_object_ids, float* host_ndc_depth, size_t num_pixels)
{
  if(!h || h->numPaths == 0 || num_pixels < (size_t)h->numPaths || (!host_object_ids && !host_ndc_depth))
    return B200PT_E_INVALID;
  if(const int rc = enter(h, false))
    return rc;
  if(host_object_ids)
    CK(cudaMemcpyAsync(host_object_ids, h->dSelect, (size_t)h->numPaths * 4, cudaMemcpyDeviceToHost, h->stream));
  if(host_ndc_depth)
    CK(cudaMemcpyAsync(host_ndc_depth, h->dNdcDepth, (size_t)h->numPaths * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return B200PT_OK;
}

int b200pt_get_selection_device(b200pt_t* h, uint32_t** dev_object_ids, float** dev_ndc_depth)
{
  if(!h || h->numPaths == 0)
    return B200PT_E_INVALID;
  if(dev_object_ids)
    *dev_object_ids = h->dSelect;
  if(dev_ndc_depth)
    *dev_ndc_depth = h->dNdcDepth;
  return B200PT_OK;
}

int b200pt_read_accum_async(b200pt_t* h, float* host, size_t num_floats, int slot)
{
  if(!h || h->numPaths == 0 || !host || num_floats < (size_t)h->numPaths * 4 || slot < 0 || slot >= 8)
    return B200PT_E_INVALID;
  if(const int rc = enter(h, false))
    return rc;
  if(!h->readDone[slot])
    CK(cudaEventCreateWithFlags(&h->readDone[slot], cudaEventDisableTiming));
  else
    CK(cudaEventSynchronize(h->readDone[slot]));
  CK(cudaMemcpyAsync(host, h->dAccum, (size_t)h->numPaths * 16, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaEventRecord(h->readDone[slot], h->stream));
  return B200PT_OK;
}

int b200pt_wait_read(b200pt_t* h, int slot)
{
  if(!h || slot < 0 || slot >= 8)
    return B200PT_E_INVALID;
  if(h->readDone[slot])
    CK(cudaEventSynchronize(h->readDone[slot]));
  return B200PT_OK;
}

// the path pool rebuilt at the current extent (interleaved or not) after a change of what it holds; an accumulation buffer the
// caller supplied (b200pt_set_accum_device) stays in use
static int rebuildPool(b200pt_t* h)
{
  if(h->numPaths == 0)
    return B200PT_OK;
  float4* const user = (h->dAccum != h->dAccumOwned) ? h->dAccum : nullptr;
  int           rc;
  if(h->bandWorld > 1)
    rc = b200pt_resize_interleaved(h, h->width, h->height, h->bandRows, h->bandWorld, h->bandRank);
  else
    rc = b200pt_resize(h, h->width, h->height, h->tileY0, h->tileRows);
  if(rc == B200PT_OK && user)
    h->dAccum = user;
  return rc;
}

int b200pt_set_frames_in_flight(b200pt_t* h, int n)
{
  if(!h || n < 1 || n > b200pt::kMaxLanes)
    return B200PT_E_INVALID;
  if(n == h->numLanes)
    return B200PT_OK;
  h->numLanes = n;
  return rebuildPool(h);
}

int b200pt_set_guide_outputs(b200pt_t* h, int enable)
{
  if(!h)
    return B200PT_E_INVALID;
  if(const int rc = enter(h, false))
    return rc;
  if((enable != 0) == h->guides)
    return B200PT_OK;
  h->guides = enable != 0;
  return rebuildPool(h);
}

int b200pt_read_guide(b200pt_t* h, float* host_albedo_normal, size_t num_floats)
{
  if(!h || h->numPaths == 0 || !h->dGuide || !host_albedo_normal || num_floats < (size_t)h->numPaths * 4)
    return B200PT_E_INVALID;
  if(const int rc = enter(h, false))
    return rc;
  CK(cudaMemcpyAsync(host_albedo_normal, h->dGuide, (size_t)h->numPaths * 16, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return B200PT_OK;
}

int b200pt_get_guide_device(b200pt_t* h, float** dev_albedo_normal, size_t* num_floats)
{
  if(!h || h->numPaths == 0 || !h->dGuide || !dev_albedo_normal)
    return B200PT_E_INVALID;
  *dev_albedo_normal = reinterpret_cast<float*>(h->dGuide);
  if(num_floats)
    *num_floats = (size_t)h->numPaths * 4;
  return B200PT_OK;
}

int b200pt_set_dlss_guides(b200pt_t* h, int enable)
{
  if(!h)
    return B200PT_E_INVALID;
  if(const int rc = enter(h, false))
    return rc;
  if((enable != 0) == h->dlss)
    return B200PT_OK;
  h->dlss = enable != 0;
  return rebuildPool(h);
}

// the six planes inside dDlss, in the order of b200pt_dlss_guides; each starts on a 256-byte boundary (dlssAllocBytes)
static void dlssPlanes(const b200pt_t* h, void* ptr[6], size_t bytes[6])
{
  const size_t n = h->numPaths;
  const size_t per[6] = {4, 8, 8, 4, 2, 2};
  size_t       off = 0;
  for(int k = 0; k < 6; k++)
  {
    ptr[k] = h->dDlss + off;
    bytes[k] = n * per[k];
    off += (bytes[k] + 255) & ~(size_t)255;
  }
}

int b200pt_read_dlss_guides(b200pt_t* h, const b200pt_dlss_guides* out)
{
  if(!h || h->numPaths == 0 || !h->dDlss || !out)
    return B200PT_E_INVALID;
  void*        dev[6];
  size_t       need[6];
  dlssPlanes(h, dev, need);
  void* const  host[6] = {out->albedo, out->spec_albedo, out->normal_roughness, out->motion, out->depth, out->spec_hit_dist};
  const size_t have[6] = {out->albedo_bytes, out->spec_albedo_bytes, out->normal_roughness_bytes, out->motion_bytes, out->depth_bytes, out->spec_hit_dist_bytes};
  for(int k = 0; k < 6; k++)
    if(host[k] && have[k] < need[k])
    {
      h->err = "b200pt_read_dlss_guides: a destination is smaller than its plane (tile_rows x width in the plane's format)";
      return B200PT_E_INVALID;
    }
  if(const int rc = enter(h, false))
    return rc;
  for(int k = 0; k < 6; k++)
    if(host[k])
      CK(cudaMemcpyAsync(host[k], dev[k], need[k], cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return B200PT_OK;
}

int b200pt_get_dlss_guides_device(b200pt_t* h, b200pt_dlss_guides* out)
{
  if(!h || h->numPaths == 0 || !h->dDlss || !out)
    return B200PT_E_INVALID;
  void*  dev[6];
  size_t bytes[6];
  dlssPlanes(h, dev, bytes);
  out->albedo = dev[0];
  out->albedo_bytes = bytes[0];
  out->spec_albedo = dev[1];
  out->spec_albedo_bytes = bytes[1];
  out->normal_roughness = dev[2];
  out->normal_roughness_bytes = bytes[2];
  out->motion = dev[3];
  out->motion_bytes = bytes[3];
  out->depth = dev[4];
  out->depth_bytes = bytes[4];
  out->spec_hit_dist = dev[5];
  out->spec_hit_dist_bytes = bytes[5];
  return B200PT_OK;
}

int b200pt_set_frame_batch(b200pt_t* h, int n)
{
  if(!h || n < 1 || n > 64)
    return B200PT_E_INVALID;
  if(n == h->batch)
    return B200PT_OK;
  if(n > 1 && h->views > 1)
  {
    h->err = "b200pt_set_frame_batch: frames are not batched while more than one view is set (b200pt_set_views)";
    return B200PT_E_UNSUPPORTED;
  }
  if(const int rc = enter(h, false))
    return rc;
  h->batch = n;
  return rebuildPool(h);
}

int b200pt_synchronize(b200pt_t* h)
{
  if(!h)
    return B200PT_E_INVALID;
  if(const int rc = enter(h, true))
    return rc;
  return checkDeviceErrors(h);
}

int b200pt_set_profiling(b200pt_t* h, int enabled)
{
  if(!h)
    return B200PT_E_INVALID;
  if(const int rc = enter(h, false))
    return rc;
  flushEvents(h);
  h->profiling = enabled != 0;
  if(h->profiling)
    CK(growEventPool(h, 2048));
  return B200PT_OK;
}

// the checks every rendered frame passes (`who` names the entry point in the error)
static int checkFrame(b200pt_t* h, const b200pt_frame_info* fi, const b200pt_push_constant* pc, const char* who)
{
  const std::string name(who);
  if(!h->haveScene || h->numPaths == 0)
  {
    h->err = name + ": set_scene and resize must come first";
    return B200PT_E_INVALID;
  }
  if(!(fi->flags & B200PT_SCENE_USE_HDR_ENVIRONMENT) || !h->haveEnv)
  {
    h->err = name + ": only the HDR environment (--envSystem 1) is built; physical sky is out of scope";
    return B200PT_E_UNSUPPORTED;
  }
  if((fi->flags & B200PT_SCENE_USE_HDR_ENVIRONMENT) && fi->envBlur > 0.0f && !(fi->flags & B200PT_SCENE_USE_SOLID_BACKGROUND))
  {
    h->err = name + ": the blurred HDR backplate (envBlur > 0: nvshaders' smoothHDRBlur, external) is not built";
    return B200PT_E_UNSUPPORTED;
  }
  if((pc->flags & B200PT_PT_USE_DLSS) && !h->dlss)
  {
    h->err = name + ": ePtUseDlss needs the DLSS guide images (b200pt_set_dlss_guides(h, 1) first)";
    return B200PT_E_INVALID;
  }
  if((pc->flags & B200PT_PT_USE_DLSS) && pc->numSamples != 1)
  {
    h->err = name + ": the DLSS variant renders one sample per frame (numSamples must be 1)";
    return B200PT_E_INVALID;
  }
  if((pc->flags & B200PT_PT_USE_OPTIX_DENOISER) && !h->guides)
  {
    h->err = name + ": ePtUseOptixDenoiser needs the guide image (b200pt_set_guide_outputs(h, 1) first)";
    return B200PT_E_INVALID;
  }
  if(pc->numSamples < 1 || pc->maxDepth < 0 || (int)fi->imageSize[0] != h->width || (int)fi->imageSize[1] != h->height)
  {
    h->err = name + ": bad numSamples / maxDepth / imageSize";
    return B200PT_E_INVALID;
  }
  return B200PT_OK;
}

int b200pt_render_frame(b200pt_t* h, const b200pt_frame_info* fi, const b200pt_push_constant* pc)
{
  if(!h || !fi || !pc)
    return B200PT_E_INVALID;
  if(const int rc = checkFrame(h, fi, pc, "b200pt_render_frame"))
    return rc;
  if(h->batch <= 1)
    return launchFrames(h, fi, pc, 1);
  if(pc->flags & B200PT_PT_USE_DLSS)
  {
    // a DLSS frame runs alone: its jitter and camera change every frame, and it replaces the image
    const int rc = flushPending(h);
    if(rc)
      return rc;
    return launchFrames(h, fi, pc, 1);
  }
  // frame batching: collect consecutive frames of a static camera (same frame constants; push constants that differ only by
  // the frame / sample counters advancing like the host loop advances them) and run them as one wavefront
  if(h->pendingCount > 0)
  {
    const b200pt_push_constant& p0 = h->pendingPc;
    b200pt_push_constant        expect = p0;
    expect.frameCount = p0.frameCount + h->pendingCount;
    expect.totalSamples = p0.totalSamples + h->pendingCount * p0.numSamples;
    expect.flags = p0.flags & ~B200PT_PT_FIRST_FRAME;
    if(memcmp(&h->pendingFi, fi, sizeof(*fi)) != 0 || memcmp(&expect, pc, sizeof(*pc)) != 0)
    {
      const int rc = flushPending(h);
      if(rc)
        return rc;
    }
  }
  if(h->pendingCount == 0)
  {
    h->pendingFi = *fi;
    h->pendingPc = *pc;
  }
  h->pendingCount++;
  if(h->pendingCount >= h->batch)
    return flushPending(h);
  return B200PT_OK;
}

int b200pt_set_views(b200pt_t* h, int n)
{
  if(!h || n < 1 || n > 64)
    return B200PT_E_INVALID;
  if(n == h->views)
    return B200PT_OK;
  if(n > 1 && h->batch > 1)
  {
    h->err = "b200pt_set_views: more than one view needs frame batching off (b200pt_set_frame_batch(h, 1))";
    return B200PT_E_UNSUPPORTED;
  }
  if(const int rc = enter(h, false))
    return rc;
  const int old = h->views;
  h->views = n;
  const int rc = rebuildPool(h);
  if(rc)
    h->views = old;  // like a failed b200pt_resize the handle has no pool now; the next resize builds it for the old count
  return rc;
}

int b200pt_render_views(b200pt_t* h, const b200pt_frame_info* fis, uint32_t n, const b200pt_push_constant* pc)
{
  if(!h || !fis || !pc)
    return B200PT_E_INVALID;
  if(n != (uint32_t)h->views)
  {
    h->err = "b200pt_render_views: n must equal the view count of b200pt_set_views";
    return B200PT_E_INVALID;
  }
  // the views share every field but the pose: fis[v] with fis[0]'s pose must be fis[0], byte for byte
  for(uint32_t v = 1; v < n; v++)
  {
    b200pt_frame_info a = fis[v];
    memcpy(a.viewMatrix, fis[0].viewMatrix, sizeof(a.viewMatrix));
    memcpy(a.viewInv, fis[0].viewInv, sizeof(a.viewInv));
    memcpy(a.viewProjMatrix, fis[0].viewProjMatrix, sizeof(a.viewProjMatrix));
    memcpy(a.prevMVP, fis[0].prevMVP, sizeof(a.prevMVP));
    if(memcmp(&a, &fis[0], sizeof(a)) != 0)
    {
      h->err = "b200pt_render_views: view " + std::to_string(v) + " differs from view 0 in a field other than viewMatrix, viewInv, viewProjMatrix and prevMVP";
      return B200PT_E_INVALID;
    }
  }
  if(n > 1 && (pc->flags & (B200PT_PT_USE_DLSS | B200PT_PT_USE_OPTIX_DENOISER)))
  {
    h->err = "b200pt_render_views: the DLSS and OptiX-denoiser guide images belong to one displayed frame; render them with b200pt_render_frame";
    return B200PT_E_UNSUPPORTED;
  }
  if(const int rc = checkFrame(h, &fis[0], pc, "b200pt_render_views"))
    return rc;
  if(const int rc = flushPending(h))
    return rc;
  return launchFrames(h, &fis[0], pc, 1, n > 1 ? fis : nullptr);
}

// view 0 is the handle's accumulation, selection and depth images; view v > 0 sits at (v - 1) x pixels in the view images
static void viewImages(b200pt_t* h, uint32_t view, float4** rgba, uint32_t** ids, float** depth)
{
  const size_t off = view ? (size_t)(view - 1) * h->numPaths : 0;
  *rgba = view ? h->dViewAccum + off : h->dAccum;
  *ids = view ? h->dViewSelect + off : h->dSelect;
  *depth = view ? h->dViewDepth + off : h->dNdcDepth;
}

int b200pt_read_views(b200pt_t* h, uint32_t view, float* host_rgba32f, uint32_t* host_object_ids, float* host_ndc_depth, size_t num_pixels)
{
  if(!h || h->numPaths == 0 || view >= (uint32_t)h->views || num_pixels < (size_t)h->numPaths)
    return B200PT_E_INVALID;
  if(const int rc = enter(h, false))
    return rc;
  float4*   rgba;
  uint32_t* ids;
  float*    depth;
  viewImages(h, view, &rgba, &ids, &depth);
  const size_t n = h->numPaths;
  if(host_rgba32f)
    CK(cudaMemcpyAsync(host_rgba32f, rgba, n * 16, cudaMemcpyDeviceToHost, h->stream));
  if(host_object_ids)
    CK(cudaMemcpyAsync(host_object_ids, ids, n * 4, cudaMemcpyDeviceToHost, h->stream));
  if(host_ndc_depth)
    CK(cudaMemcpyAsync(host_ndc_depth, depth, n * 4, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return B200PT_OK;
}

int b200pt_get_views_device(b200pt_t* h, uint32_t view, float** dev_rgba32f, uint32_t** dev_object_ids, float** dev_ndc_depth)
{
  if(!h || h->numPaths == 0 || view >= (uint32_t)h->views)
    return B200PT_E_INVALID;
  float4*   rgba;
  uint32_t* ids;
  float*    depth;
  viewImages(h, view, &rgba, &ids, &depth);
  if(dev_rgba32f)
    *dev_rgba32f = reinterpret_cast<float*>(rgba);
  if(dev_object_ids)
    *dev_object_ids = ids;
  if(dev_ndc_depth)
    *dev_ndc_depth = depth;
  return B200PT_OK;
}

static int flushPending(b200pt_t* h)
{
  if(h->pendingCount == 0)
    return B200PT_OK;
  const int n = h->pendingCount;
  h->pendingCount = 0;
  return launchFrames(h, &h->pendingFi, &h->pendingPc, n);
}

int b200pt_flush(b200pt_t* h)
{
  if(!h)
    return B200PT_E_INVALID;
  return flushPending(h);
}

// enqueues the launch chain of `count` consecutive frames (count > 1: one batched wavefront, FrameParams::batch), or with viewFis
// (count 1) of the handle's views, whose poses replace fi's (FrameParams::views)
static int launchFrames(b200pt_t* h, const b200pt_frame_info* fi, const b200pt_push_constant* pc, int count, const b200pt_frame_info* viewFis)
{
  CK(cudaSetDevice(h->device));
  FrameParams F;
  F.fi = *fi;
  F.pc = *pc;
  F.width = h->width;
  F.height = h->height;
  F.tileY0 = h->tileY0;
  F.tileRows = h->tileRows;
  F.bandRows = h->bandRows;
  F.bandWorld = h->bandWorld;
  F.bandRank = h->bandRank;
  F.pixels = h->numPaths;
  F.batch = count;
  F.views = viewFis ? h->views : 1;
  F.poses = nullptr;
  F.numPaths = h->numPaths * (uint32_t)count * (uint32_t)F.views;
  F.prevObjectToWorld = ((pc->flags & B200PT_PT_USE_DLSS) && h->prevO2WValid) ? h->dPrevO2W : nullptr;
  h->prevO2WValid = false;
  h->renderedSinceUpdate = true;

  const int     laneIdx = (int)(h->frameSerial++ % (uint64_t)h->numLanes);
  b200pt::Lane& L = h->lanes[laneIdx];
  // the lane's pool is free once the accumulate of its previous frame ran; while profiling, frames are serialised
  // (wait for the previous frame's accumulate) so per-kernel event times are not inflated by overlap
  if(L.busy)
    CK(cudaStreamWaitEvent(L.stream, L.freed, 0));
  if(h->profiling && h->lastLane >= 0 && h->lastLane != laneIdx)
    CK(cudaStreamWaitEvent(L.stream, h->lanes[h->lastLane].freed, 0));
  if(F.views > 1)
  {
    // on the lane's stream, behind the wait: the lane's previous frame has read its poses
    std::vector<ViewPose> poses((size_t)F.views);
    for(int v = 0; v < F.views; v++)
    {
      memcpy(poses[v].viewMatrix, viewFis[v].viewMatrix, sizeof(poses[v].viewMatrix));
      memcpy(poses[v].viewInv, viewFis[v].viewInv, sizeof(poses[v].viewInv));
      memcpy(poses[v].viewProjMatrix, viewFis[v].viewProjMatrix, sizeof(poses[v].viewProjMatrix));
      memcpy(poses[v].prevMVP, viewFis[v].prevMVP, sizeof(poses[v].prevMVP));
    }
    CK(cudaMemcpyAsync(L.poses, poses.data(), poses.size() * sizeof(ViewPose), cudaMemcpyHostToDevice, L.stream));
    F.poses = L.poses;
  }
  const Counters C{L.dCounters, kMaxIters};
  CK(cudaMemsetAsync(L.dCounters, 0, sizeof(uint32_t) * kCounterArrays * kMaxIters, L.stream));
  Launcher ctx{h, L.stream, laneIdx, h->frameSerial - 1, -1, h->profiling || h->timeline != nullptr, F.numPaths};
  const int gridWide = gridFor(h, 8);
  ctx(kStageOther, [&](cudaStream_t st) { k_raygen<<<gridWide, 256, 0, st>>>(L.P, F, L.dQ[0], C.trace(0), h->dStats); });

  int it = 0;  // bounces run
  if(pc->maxDepth > 0)
  {
    const int gS = gridFor(h, kShadeCtasPerSM);  // persistent shade kernel
    const uint32_t feat = shadeFeatures(h);
    const auto     shade = feat == 0u ? k_shade<0u> : feat == FEAT_LEAN ? k_shade<FEAT_LEAN> : k_shade<FEAT_ALL>;
    const bool        sortShade = h->sortShade && h->S.numMaterials + 1 <= kSortMaxBuckets;
    int               cur = 0;  // dQ[cur] = trace queue, dQ[2] = post queue, dQ[1-cur] = next queue
    // (a shadowed shadow-catcher hit continues without consuming depth: such a frame can need more iterations than maxDepth)
    const bool catcherFrame = (fi->flags & B200PT_SCENE_USE_INFINITE_PLANE) && (fi->flags & B200PT_SCENE_INFINITE_PLANE_SHADOW_CATCHER);
    const bool mayOverrun = h->hasVolume || pc->numSamples > 1 || catcherFrame;
    int        remaining = pc->maxDepth;
    for(;;)
    {
      for(int k = 0; k < remaining && it < kMaxIters - 1; k++, it++)
      {
        ctx.bounce = it;
        uint32_t*       qT = L.dQ[cur];
        uint32_t*       qN = L.dQ[1 - cur];
        launchWalk(ctx, 0, L.P, qT, L.dQ[4], L.dQ[5], C, it, 0);
        const uint32_t* qShade = qT;
        if(sortShade)
        {
          // dQ[4] (the any-hit queue) is free between the closest-hit any-hit kernels and the shadow walk
          launchSort(ctx, L, qT, C.trace(it), L.dQ[4], (uint32_t)h->S.numMaterials + 1u);
          qShade = L.dQ[4];
        }
        ctx(kStageShade, [&](cudaStream_t st) {
          shade<<<gS, kShadeBlock, 2048, st>>>(L.P, h->S, F, qShade, C.trace(it), L.dQ[2], C.post(it), L.dQ[3], C.shadow(it), qN, C.trace(it + 1), h->dStats);
        });
        launchWalk(ctx, 1, L.P, L.dQ[3], L.dQ[4], L.dQ[5], C, it, 0);
        ctx(kStageResolve, [&](cudaStream_t st) { k_resolve<<<gridFor(h, 4), 256, 0, st>>>(L.P, h->S, F, L.dQ[2], C.post(it), qN, C.trace(it + 1), h->dStats); });
        cur = 1 - cur;
      }
      if(!mayOverrun)
        break;
      CK(cudaMemcpyAsync(L.hCount, C.trace(it), sizeof(uint32_t), cudaMemcpyDeviceToHost, L.stream));
      CK(cudaStreamSynchronize(L.stream));
      if(L.hCount[0] == 0)
        break;
      if(it >= kMaxIters - 1)
      {
        h->err = "b200pt_render_frame: iteration budget exhausted (runaway volume walk?)";
        return B200PT_E_INVALID;
      }
      remaining = 4;
    }
    ctx.bounce = -1;
  }
  // accumulate on the main stream, in frame order
  CK(cudaEventRecord(L.done, L.stream));
  CK(cudaStreamWaitEvent(h->stream, L.done, 0));
  ctx.stream = h->stream;
  ctx.lane = -1;
  if(pc->flags & B200PT_PT_FIRST_FRAME)
    ctx(kStageOther, [&](cudaStream_t st) { k_select<<<gridWide, 128, 0, st>>>(h->S, F, h->dSelect, h->dViewSelect, h->dStats); });
  ctx(kStageOther, [&](cudaStream_t st) { k_accumulate<<<gridWide, 256, 0, st>>>(L.P, F, h->dAccum, h->dNdcDepth, h->dViewAccum, h->dViewDepth); });
  if((pc->flags & B200PT_PT_USE_OPTIX_DENOISER) && h->dGuide)
    ctx(kStageOther, [&](cudaStream_t st) { k_guide<<<gridWide, 256, 0, st>>>(L.P, F, h->dGuide); });
  if((pc->flags & B200PT_PT_USE_DLSS) && h->dDlss)
  {
    void*  dev[6];
    size_t bytes[6];
    dlssPlanes(h, dev, bytes);
    const DlssPlanes planes{(uint32_t*)dev[0], (uint2*)dev[1], (uint2*)dev[2], (uint32_t*)dev[3], (uint16_t*)dev[4], (uint16_t*)dev[5]};
    ctx(kStageOther, [&](cudaStream_t st) { k_dlss_guides<<<gridWide, 256, 0, st>>>(L.P, F, planes); });
  }
  CK(cudaEventRecord(L.freed, h->stream));
  L.busy = true;
  h->lastLane = laneIdx;
  CK(cudaGetLastError());
  if(h->profiling && getenv("B200PT_DUMP_ITERS"))
  {
    // tuning aid: this frame's queue sizes and per-stage kernel times of every bounce it ran, from the events tagged with the frame and
    // bounce, then the launches outside the bounce loop (stderr; events of the frame that a full pool flushed early are missing)
    CK(cudaStreamSynchronize(h->stream));
    std::vector<uint32_t> c((size_t)kCounterArrays * kMaxIters);
    CK(cudaMemcpy(c.data(), L.dCounters, sizeof(uint32_t) * c.size(), cudaMemcpyDeviceToHost));
    const Counters      hc{c.data(), kMaxIters};
    std::vector<double> ms((size_t)(it + 1) * kStageCount, 0.0);  // [bounce][stage]; bounce `it`: outside the bounce loop
    for(size_t e = 0; e < h->evUsed; e++)
    {
      const b200pt::EvRec& r = h->evPool[e];
      float                t = 0.f;
      if(r.frame == ctx.frame && cudaEventElapsedTime(&t, r.a, r.b) == cudaSuccess)
        ms[(size_t)(r.bounce < 0 ? it : r.bounce) * kStageCount + r.cat] += t;
    }
    for(int b = 0; b < it; b++)
    {
      const double* m = &ms[(size_t)b * kStageCount];
      fprintf(stderr, "iter %2d  %8u rays  k_trace %.3f  k_alpha %.3f  k_shade %.3f | %8u shadow rays  k_shadow %.3f | %8u paths  k_resolve %.3f | other %.3f ms\n", b,
                *hc.trace(b), m[kStageTrace], m[kStageAnyHit], m[kStageShade], *hc.shadow(b), m[kStageShadow], *hc.post(b), m[kStageResolve], m[kStageOther]);
      // any-hit rounds: paths entering k_alpha in round r and paths sent on to continuation round r
      for(int kind = 0; kind < 2; kind++)
      {
        fprintf(stderr, "         %s any-hit", kind ? "shadow " : "closest");
        for(int r = 0; r <= h->contRounds; r++)
          fprintf(stderr, " %u%s", *hc.anyHit(kind, r, b), r < h->contRounds ? "" : "\n");
        fprintf(stderr, "         %s cont   ", kind ? "shadow " : "closest");
        for(int r = 0; r < h->contRounds; r++)
          fprintf(stderr, " %u", *hc.cont(kind, r, b));
        fprintf(stderr, "\n");
      }
    }
    fprintf(stderr, "outside the bounce loop: other %.3f ms\n", ms[(size_t)it * kStageCount + kStageOther]);
  }
  return B200PT_OK;
}

int b200pt_get_stats(b200pt_t* h, b200pt_stats* out)
{
  if(!h || !out)
    return B200PT_E_INVALID;
  if(const int rc = enter(h, true))
    return rc;
  DevStats d{};
  CK(cudaMemcpy(&d, h->dStats, sizeof(d), cudaMemcpyDeviceToHost));
  out->closestRays = d.closestRays;
  out->shadowRays = d.shadowRays;
  out->shadedHits = d.shadedHits;
  out->pathsStarted = d.pathsStarted;
  out->nodesVisited = d.nodesVisited;
  out->trisTested = d.trisTested;
#ifdef B200PT_COUNT_TRAVERSAL
  if(getenv("B200PT_DUMP_ITERS") && d.warpIters)
    fprintf(stderr, "traversal loop: %llu warp iterations, busy lanes %.2f/32, node-phase lanes %.2f/32, triangle-phase lanes %.2f/32\n", d.warpIters,
            (double)d.busyLaneIters / (double)d.warpIters, (double)d.nodesVisited / (double)d.warpIters, (double)d.trisTested / (double)d.warpIters);
#endif
  flushEvents(h);
  out->msTraceClosest = h->msCat[kStageTrace];
  out->msShade = h->msCat[kStageShade];
  out->msTraceShadow = h->msCat[kStageShadow];
  out->msOther = h->msCat[kStageOther];
  out->msAnyHit = h->msCat[kStageAnyHit];
  out->msResolve = h->msCat[kStageResolve];
  out->msTotal = std::accumulate(std::begin(h->msCat), std::end(h->msCat), 0.0);
  out->kernelLaunches = h->kernelLaunches;
  out->launchesTraceClosest = h->launchesCat[kStageTrace];
  out->launchesShade = h->launchesCat[kStageShade];
  out->launchesTraceShadow = h->launchesCat[kStageShadow];
  out->launchesAnyHit = h->launchesCat[kStageAnyHit];
  out->launchesResolve = h->launchesCat[kStageResolve];
  return B200PT_OK;
}

int b200pt_reset_stats(b200pt_t* h)
{
  if(!h)
    return B200PT_E_INVALID;
  if(const int rc = enter(h, true))
    return rc;
  CK(cudaMemset(h->dStats, 0, sizeof(DevStats)));
  flushEvents(h);
  std::fill(std::begin(h->msCat), std::end(h->msCat), 0.0);
  std::fill(std::begin(h->launchesCat), std::end(h->launchesCat), 0);
  h->kernelLaunches = 0;
  return B200PT_OK;
}

// ray-level API: the rays run through the walk sequence of a frame's bounce (launchWalk: the same kernels, continuation rounds and grid
// rule) on a scratch pool, so the ray-level parity tests check what frames run
static int ensureRayPool(b200pt_t* h, uint32_t n)
{
  if(n <= h->rayCapacity)
    return B200PT_OK;
  syncAll(h);
  freeRayPool(h);
  DeviceArena A;
  PathState   P;
  allocPathState(h, A, n, P);
  uint32_t* const q[3] = {A.alloc<uint32_t>(n), A.alloc<uint32_t>(n), A.alloc<uint32_t>(n)};
  uint32_t* const counters = A.alloc<uint32_t>(kCounterArrays);
  if(!A.ok())
    return failed(h, A, "ray-level API");
  h->rayMem = std::move(A);
  h->rayP = P;
  std::copy(q, q + 3, h->rayQ);
  h->rayCounters = counters;
  h->rayCapacity = n;
  return B200PT_OK;
}

// the walk of n rays (records of recordFloats floats, the ray first) into the ray pool; the caller reads the pool out
static int walkRays(b200pt_t* h, const float* dev_rays, uint32_t recordFloats, uint32_t n, uint32_t* dev_seeds, int shadow, const Launcher& ctx)
{
  const int rc = ensureRayPool(h, n);
  if(rc)
    return rc;
  const Counters C{h->rayCounters, 1};
  CK(cudaMemsetAsync(h->rayCounters, 0, sizeof(uint32_t) * kCounterArrays, h->stream));
  ctx(kStageOther, [&](cudaStream_t st) {
    k_rays_load<<<gridFor(h, 8), 256, 0, st>>>(h->rayP, reinterpret_cast<const float4*>(dev_rays), recordFloats / 4, n, dev_seeds, h->rayQ[0],
                                               C.queue(shadow, 0), shadow);
  });
  launchWalk(ctx, shadow, h->rayP, h->rayQ[0], h->rayQ[1], h->rayQ[2], C, 0, shadow ? 0 : TRACE_TMIN);
  return B200PT_OK;
}

static int traceRays(b200pt_t* h, const float* dev_rays, uint32_t n, float* dev_out, uint32_t* dev_seeds, int shadow)
{
  if(!h || !h->haveScene || !dev_rays || !dev_out)
    return B200PT_E_INVALID;
  CK(cudaSetDevice(h->device));
  if(n == 0)
    return B200PT_OK;
  const Launcher ctx{h, h->stream, -1, 0, -1, false, n};
  if(const int rc = walkRays(h, dev_rays, 8, n, dev_seeds, shadow, ctx))
    return rc;
  ctx(kStageOther, [&](cudaStream_t st) { k_rays_store<<<gridFor(h, 8), 256, 0, st>>>(h->rayP, h->S, n, dev_out, dev_seeds, shadow); });
  CK(cudaGetLastError());
  return B200PT_OK;
}

int b200pt_trace_closest(b200pt_t* h, const float* dev_rays, uint32_t n, float* dev_hits, uint32_t* dev_seeds)
{
  return traceRays(h, dev_rays, n, dev_hits, dev_seeds, 0);
}

int b200pt_trace_shadow(b200pt_t* h, const float* dev_rays, uint32_t n, float* dev_transmission, uint32_t* dev_seeds)
{
  return traceRays(h, dev_rays, n, dev_transmission, dev_seeds, 1);
}

int b200pt_shade_state(b200pt_t* h, const float* dev_in, uint32_t n, float* dev_out, uint32_t* dev_seeds)
{
  if(!h)
    return B200PT_E_INVALID;
  if(!dev_in || !dev_out || !h->haveScene)
  {
    h->err = "b200pt_shade_state: needs a scene and device buffers";
    return B200PT_E_INVALID;
  }
  CK(cudaSetDevice(h->device));
  if(n == 0)
    return B200PT_OK;
  const Launcher ctx{h, h->stream, -1, 0, -1, false, n};
  if(const int rc = walkRays(h, dev_in, 16, n, dev_seeds, 0, ctx))
    return rc;
  const uint32_t feat = shadeFeatures(h);
  const auto     shade = feat == 0u ? k_shade_state<0u> : feat == FEAT_LEAN ? k_shade_state<FEAT_LEAN> : k_shade_state<FEAT_ALL>;
  ctx(kStageOther, [&](cudaStream_t st) { shade<<<(n + 127) / 128, 128, 2048, st>>>(h->rayP, h->S, dev_in, n, dev_out, dev_seeds); });
  CK(cudaGetLastError());
  return B200PT_OK;
}

int b200pt_bsdf_eval(b200pt_t* h, const float* dev_in, uint32_t n, float* dev_out)
{
  if(!h || !dev_in || !dev_out)
    return B200PT_E_INVALID;
  CK(cudaSetDevice(h->device));
  if(n)
    k_bsdf_eval<<<(n + 127) / 128, 128, 0, h->stream>>>(dev_in, n, dev_out);
  CK(cudaGetLastError());
  return B200PT_OK;
}

int b200pt_bsdf_sample(b200pt_t* h, const float* dev_in, uint32_t n, float* dev_out)
{
  if(!h || !dev_in || !dev_out)
    return B200PT_E_INVALID;
  CK(cudaSetDevice(h->device));
  if(n)
    k_bsdf_sample<<<(n + 127) / 128, 128, 0, h->stream>>>(dev_in, n, dev_out);
  CK(cudaGetLastError());
  return B200PT_OK;
}

int b200pt_texture_lookup(b200pt_t* h, const float* dev_in, uint32_t n, float* dev_out)
{
  if(!h)
    return B200PT_E_INVALID;
  if(!dev_in || !dev_out || !h->haveScene)
  {
    h->err = "b200pt_texture_lookup: needs a scene and device buffers";
    return B200PT_E_INVALID;
  }
  CK(cudaSetDevice(h->device));
  if(!n)
    return B200PT_OK;
  // the records are validated on the host: a slot beyond the scene's texture infos would read past S.texInfos
  std::vector<float> rec((size_t)n * 8);
  CK(cudaMemcpy(rec.data(), dev_in, rec.size() * sizeof(float), cudaMemcpyDeviceToHost));
  for(uint32_t i = 0; i < n; i++)
  {
    const float slot = rec[(size_t)i * 8], mode = rec[(size_t)i * 8 + 1];
    if(!(slot >= 0.0f && slot < (float)h->numTextureInfos && slot == floorf(slot)) || !(mode == 0.0f || mode == 1.0f))
    {
      h->err = "b200pt_texture_lookup: record " + std::to_string(i) + " has a texture-info slot outside the scene or a mode other than 0 / 1";
      return B200PT_E_INVALID;
    }
  }
  k_texture_lookup<<<(n + 127) / 128, 128, 2048, h->stream>>>(h->S, dev_in, n, dev_out);
  CK(cudaGetLastError());
  return B200PT_OK;
}

}  // extern "C"
