// dlss_oracle.cpp — the DLSS variant of the CPU oracle (TEST INFRASTRUCTURE, loaded by tests/dlss_oracle.py only).
//
// The path tracer's DLSS variant (PathtracerFlags::ePtUseDlss; shaders/dlss_util.h, shaders/gltf_pathtrace.slang:135-143, 216-263,
// 370-377, 564-651, shaders/pathtrace_functions.h.slang:65-102, 942-988) restated on top of the scalar fp32 oracle: this file
// includes oracle/pt_oracle.cpp for the shared arithmetic (traversal, getHitState, evaluateMaterial, lights, BSDFs, volumes) and
// restates the parts the variant changes -- pathTraceOneBounce with the DLSS captures, pathTrace, samplePixel and processPixel with
// the frame jitter, the replaced image and the six guide images -- independently of the device sources (csrc/dlss_guides.cuh).
// Built like the oracle (-ffp-contract=off) into its own shared library, which also exports the oracle's own entry points.
#include "../oracle/pt_oracle.cpp"

#include <cstring>

namespace dlss_variant {

// per-frame context of a DLSS frame
struct DlssCtx : Ctx
{
  const float* prevObjectToWorld;  // previous-frame objectToWorld per render node (16 floats, glm order), or null: camera-only motion
};

// PathTracerState + the USE_DLSS_SHADER fields (GuideScratch, pathtrace_functions.h.slang:79-88; firstHitPosPrev)
struct PathState : PathTracerState
{
  float  guideRoughness = 0.0f;
  float3 firstHitPosPrev = f3(1e34f);  // previous-frame position of the first hit
  float3 specAlbedo = f3(0.0f);        // GuideScratch::specularAlbedo (float16_t)
  float  specHitDist = 0.0f;           // GuideScratch::specularHitDist (float16_t)
  bool   captureSpecularHit = false;
};

static inline uint16_t halfBits(float x)
{
  const _Float16 h = (_Float16)x;
  uint16_t       b;
  memcpy(&b, &h, 2);
  return b;
}

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

// pathTraceOneBounce (gltf_pathtrace.slang:87-430) of the DLSS variant: the oracle's restatement with the USE_DLSS_SHADER captures
static PathStepResult pathTraceOneBounce(const DlssCtx& c, Ray& ray, uint32_t& seed, PathState& pt, BounceScratch& bounce)
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
    // USE_GUIDE_SHADER (gltf_pathtrace.slang:240-263): base colour, shading normal and roughness of the first hit, stored as
    // float16_t by the reference
    pt.guideAlbedo = f3(half16(pbrMat.baseColor.x), half16(pbrMat.baseColor.y), half16(pbrMat.baseColor.z));
    pt.guideNormal = f3(half16(pbrMat.N.x), half16(pbrMat.N.y), half16(pbrMat.N.z));
    pt.guideRoughness = half16(pbrMat.roughness.x);
    {
      // instance motion (:235-241): the surface point in object space, then through the previous frame's objectToWorld
      pt.firstHitPosPrev = hit.pos;
      if(!hitInfinitePlane && c.prevObjectToWorld)
      {
        const float4 objPos = mul_vM(f4(hit.pos.x, hit.pos.y, hit.pos.z, 1.0f), *(const mat4*)o.nodes[payload.rnodeID].worldToObject);
        pt.firstHitPosPrev = xyz(mul_vM(f4(objPos.x, objPos.y, objPos.z, 1.0f), *(const mat4*)(c.prevObjectToWorld + 16 * (size_t)payload.rnodeID)));
      }
      // specular albedo (:246-255); pow(x, 2.0) is the correctly rounded square
      const float  q = (pbrMat.ior2 - pbrMat.ior1) / (pbrMat.ior2 + pbrMat.ior1);
      const float  f0FromIor = q * q;
      const float3 clamped = f3(fminf(f0FromIor * pbrMat.specularColor.x, 1.0f), fminf(f0FromIor * pbrMat.specularColor.y, 1.0f),
                                fminf(f0FromIor * pbrMat.specularColor.z, 1.0f));
      const float3 sa = envBRDFApprox2(clamped, pbrMat.roughness.x, dot(pbrMat.N, ray.d));
      pt.specAlbedo = f3(half16(sa.x), half16(sa.y), half16(sa.z));
    }
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
    if(firstRay && (sd.event_type == BSDF_EVENT_GLOSSY_REFLECTION || sd.event_type == BSDF_EVENT_IMPULSE_REFLECTION))
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
  float  guideRoughness;
  float3 hitPositionPrev, specAlbedo;
  float  specHitDist;
};

static SampleResult pathTrace(const DlssCtx& c, Ray ray, uint32_t& seed)
{
  PathState pt;
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

static SampleResult samplePixel(const DlssCtx& c, uint32_t& seed, float2 samplePos, float2 jitter, float2 imageSize)
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

struct DlssOut
{
  uint32_t* albedo;       // RGBA8 UNORM
  uint16_t* specAlbedo;   // RGBA16F
  uint16_t* normalRough;  // RGBA16F
  uint16_t* motion;       // RG16F
  uint16_t* depth;        // R16F
  uint16_t* specHitDist;  // R16F
};
static uint32_t unorm8(float x) { return (uint32_t)roundf(fminf(fmaxf(x, 0.0f), 1.0f) * 255.0f); }

// processPixel (gltf_pathtrace.slang:546-651) of the DLSS variant: one sample (the sample loop is compiled out), the image replaced
static void processPixel(const DlssCtx& c, int x, int y, float* px, uint32_t* objectId, float* ndcDepth, float* guide, const DlssOut* dlss)
{
  const float2 imageSize = f2(c.fi->imageSize[0], c.fi->imageSize[1]);
  const float2 samplePos = f2((float)x, (float)y);
  uint32_t     seed = xxhash32((uint32_t)x, (uint32_t)y, (uint32_t)c.pc->frameCount);
  dbgPixel = ((float)x == c.pc->mouseCoord[0] && (float)y == c.pc->mouseCoord[1]);
  const bool   firstFrame = (c.pc->flags & B200PT_PT_FIRST_FRAME) != 0;
  // the frame's DLSS jitter; no Gaussian draw (gltf_pathtrace.slang:568-572)
  const float2 jitter = f2(0.5f + c.fi->jitter[0], 0.5f + c.fi->jitter[1]);
  tls.paths++;
  SampleResult sr = samplePixel(c, seed, samplePos, jitter, imageSize);
  const float4 pixelColor = sr.radiance;
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
  px[0] = pixelColor.x;
  px[1] = pixelColor.y;
  px[2] = pixelColor.z;
  px[3] = pixelColor.w;
}

}  // namespace dlss_variant

extern "C" {

// A frame of the DLSS variant (refused unless pc carries B200PT_PT_USE_DLSS, with numSamples == 1 and the planes).  dlssPlanes: six pointers
// to the tile's planes (rows x width each): albedo RGBA8, specular albedo RGBA16F, normal / roughness RGBA16F, motion RG16F, depth
// R16F, specular hit distance R16F.  prevObjectToWorld: 16 floats per render node (the previous frame's objectToWorld), or null for
// camera-only motion.
int oracle_render_frame_dlss(void* h, const b200pt_frame_info* fi, const b200pt_push_constant* pc, float* accum, uint32_t* objectId, float* ndcDepth, float* guide,
                             const float* prevObjectToWorld, void* const* dlssPlanes, int y0, int rows, int nthreads)
{
  Oracle& o = *(Oracle*)h;
  if(!(fi->flags & B200PT_SCENE_USE_HDR_ENVIRONMENT) || o.envW == 0)
    return B200PT_E_UNSUPPORTED;
  if(fi->envBlur > 0.0f && !(fi->flags & B200PT_SCENE_USE_SOLID_BACKGROUND))
    return B200PT_E_UNSUPPORTED;  // tryPrimaryMissBackplate's smoothHDRBlur (nvshaders, external)
  if(!(pc->flags & B200PT_PT_USE_DLSS) || !dlssPlanes || pc->numSamples != 1)
    return B200PT_E_INVALID;
  const dlss_variant::DlssCtx c{{&o, fi, pc}, prevObjectToWorld};
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
        const size_t p = (size_t)r * W + x;
        const dlss_variant::DlssOut d{(uint32_t*)dlssPlanes[0] + p, (uint16_t*)dlssPlanes[1] + 4 * p, (uint16_t*)dlssPlanes[2] + 4 * p,
                                      (uint16_t*)dlssPlanes[3] + 2 * p, (uint16_t*)dlssPlanes[4] + p, (uint16_t*)dlssPlanes[5] + p};
        dlss_variant::processPixel(c, x, y0 + r, accum + p * 4, objectId ? objectId + p : nullptr, ndcDepth ? ndcDepth + p : nullptr,
                                   guide ? guide + p * 4 : nullptr, &d);
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

// DLSS arithmetic on records, for the tests: EnvBRDFApprox2 on (specular colour xyz, alpha, NoV) -> rgb; calculateMotionVector on
// (current xyzw, previous xyzw, resolution xy) with the two view-projection matrices (glm order) -> pixel motion xy
int oracle_env_brdf_approx2(const float* in, uint32_t n, float* out)
{
  for(uint32_t i = 0; i < n; i++)
  {
    const float* p = in + 5 * (size_t)i;
    const float3 r = dlss_variant::envBRDFApprox2(f3(p[0], p[1], p[2]), p[3], p[4]);
    out[3 * i + 0] = r.x;
    out[3 * i + 1] = r.y;
    out[3 * i + 2] = r.z;
  }
  return 0;
}
int oracle_motion_vector(const float* in, uint32_t n, const float* prevMVP, const float* currMVP, float* out)
{
  for(uint32_t i = 0; i < n; i++)
  {
    const float* p = in + 10 * (size_t)i;
    const float2 mv = dlss_variant::calculateMotionVector(f4(p[0], p[1], p[2], p[3]), f4(p[4], p[5], p[6], p[7]), *(const mat4*)prevMVP, *(const mat4*)currMVP, f2(p[8], p[9]));
    out[2 * i + 0] = mv.x;
    out[2 * i + 1] = mv.y;
  }
  return 0;
}

}  // extern "C"
