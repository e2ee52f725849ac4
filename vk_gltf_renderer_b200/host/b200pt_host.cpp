// b200pt_host.cpp — see b200pt_host.hpp.
#include "b200pt_host.hpp"

#include <cmath>
#include <cstdio>
#include <cstring>
#include <fstream>

namespace b200host {

// ------------------------------------------------------------------------------------------------
// scene blob
// ------------------------------------------------------------------------------------------------
namespace {

struct Reader
{
  std::ifstream f;
  explicit Reader(const std::string& path)
      : f(path, std::ios::binary)
  {
    if(!f)
      throw Error("cannot open scene blob " + path);
  }
  bool tryRaw(void* dst, size_t bytes)  // false at a clean end of file
  {
    f.read(static_cast<char*>(dst), (std::streamsize)bytes);
    if(f.gcount() == 0)
      return false;
    if((size_t)f.gcount() != bytes)
      throw Error("scene blob truncated");
    return true;
  }
  void raw(void* dst, size_t bytes)
  {
    f.read(static_cast<char*>(dst), (std::streamsize)bytes);
    if((size_t)f.gcount() != bytes)
      throw Error("scene blob truncated");
  }
  template <typename T>
  T pod()
  {
    T v;
    raw(&v, sizeof(T));
    return v;
  }
  template <typename T>
  void vec(std::vector<T>& v, size_t n)
  {
    v.resize(n);
    if(n)
      raw(v.data(), n * sizeof(T));
  }
};

}  // namespace

void SceneData::load(const std::string& path)
{
  Reader r(path);
  char   magic[4];
  r.raw(magic, 4);
  if(std::memcmp(magic, "B2SC", 4) != 0)
    throw Error("not a B2SC scene blob: " + path);
  const uint32_t version = r.pod<uint32_t>();
  if(version != 1)
    throw Error("unsupported scene blob version");
  const uint32_t nNodes = r.pod<uint32_t>(), nPrims = r.pod<uint32_t>(), nMats = r.pod<uint32_t>(), nInfos = r.pod<uint32_t>(),
                 nTex = r.pod<uint32_t>(), nLights = r.pod<uint32_t>();
  camera.orthographic = r.pod<uint32_t>() != 0;
  float c[14];
  r.raw(c, sizeof(c));
  std::memcpy(camera.eye, c, 12);
  std::memcpy(camera.center, c + 3, 12);
  std::memcpy(camera.up, c + 6, 12);
  camera.yfov = c[9];
  camera.znear = c[10];
  camera.zfar = c[11];
  camera.xmag = c[12];
  camera.ymag = c[13];

  m_nodes.assign(nNodes, b200pt_render_node{});
  m_visible.assign(nNodes, 1);
  for(uint32_t i = 0; i < nNodes; i++)
  {
    r.raw(m_nodes[i].objectToWorld, 64);
    r.raw(m_nodes[i].worldToObject, 64);
    m_nodes[i].materialID = r.pod<int32_t>();
    m_nodes[i].renderPrimID = r.pod<int32_t>();
    m_visible[i] = r.pod<uint32_t>() ? 1 : 0;
  }
  m_primData.assign(nPrims, Prim{});
  m_prims.assign(nPrims, b200pt_render_primitive{});
  for(uint32_t i = 0; i < nPrims; i++)
  {
    Prim&          p = m_primData[i];
    const uint32_t vc = r.pod<uint32_t>(), tc = r.pod<uint32_t>(), mask = r.pod<uint32_t>();
    r.vec(p.positions, (size_t)vc * 3);
    r.vec(p.indices, (size_t)tc * 3);
    if(mask & 1u)
      r.vec(p.normals, (size_t)vc * 3);
    if(mask & 2u)
      r.vec(p.uv0, (size_t)vc * 2);
    if(mask & 4u)
      r.vec(p.uv1, (size_t)vc * 2);
    if(mask & 8u)
      r.vec(p.tangents, (size_t)vc * 4);
    if(mask & 16u)
      r.vec(p.colors, (size_t)vc);
    b200pt_render_primitive& d = m_prims[i];
    d.indices = p.indices.data();
    d.positions = p.positions.data();
    d.normals = p.normals.empty() ? nullptr : p.normals.data();
    d.colors = p.colors.empty() ? nullptr : p.colors.data();
    d.tangents = p.tangents.empty() ? nullptr : p.tangents.data();
    d.texCoords[0] = p.uv0.empty() ? nullptr : p.uv0.data();
    d.texCoords[1] = p.uv1.empty() ? nullptr : p.uv1.data();
    d.triangleCount = tc;
    d.vertexCount = vc;
  }
  r.vec(m_materials, nMats);
  r.vec(m_texInfos, nInfos);
  m_texPixels.assign(nTex, {});
  m_textures.assign(nTex, b200pt_texture{});
  for(uint32_t i = 0; i < nTex; i++)
  {
    int32_t h[7];
    r.raw(h, sizeof(h));
    r.vec(m_texPixels[i], (size_t)h[0] * (size_t)h[1] * 4);
    b200pt_texture& t = m_textures[i];
    t.rgba8 = m_texPixels[i].data();
    t.width = h[0];
    t.height = h[1];
    t.srgb = h[2];
    t.wrapS = h[3];
    t.wrapT = h[4];
    t.magFilter = h[5];
    t.minFilter = h[6];
  }
  r.vec(m_lights, nLights);
  hdrWidth = (int)r.pod<uint32_t>();
  hdrHeight = (int)r.pod<uint32_t>();
  r.vec(hdrRgb, (size_t)hdrWidth * (size_t)hdrHeight * 3);
  // optional: the asset's EXT_mesh_opacity_micromap arrays (what SceneOmm::create uploads, src/gltf_scene_omm.cpp)
  m_ommData.clear();
  m_ommTris.clear();
  m_ommIdx.clear();
  m_micromaps.clear();
  m_primOmms.clear();
  char tag[4];
  if(r.tryRaw(tag, 4))
  {
    if(std::memcmp(tag, "OMM1", 4) != 0)
      throw Error("unknown trailing section in scene blob");
    const uint32_t nMm = r.pod<uint32_t>(), nLinks = r.pod<uint32_t>();
    m_ommData.resize(nMm);
    m_ommTris.resize(nMm);
    m_micromaps.assign(nMm, b200pt_micromap{});
    for(uint32_t i = 0; i < nMm; i++)
    {
      const uint64_t nData = r.pod<uint64_t>();
      const uint32_t nTris = r.pod<uint32_t>();
      r.vec(m_ommData[i], (size_t)nData);
      r.vec(m_ommTris[i], nTris);
      m_micromaps[i] = b200pt_micromap{m_ommData[i].data(), nData, m_ommTris[i].data(), nTris};
    }
    m_ommIdx.resize(nLinks);
    m_primOmms.assign(nLinks, b200pt_primitive_omm{});
    for(uint32_t i = 0; i < nLinks; i++)
    {
      uint32_t h[4];
      r.raw(h, sizeof(h));
      r.vec(m_ommIdx[i], h[3]);
      m_primOmms[i] = b200pt_primitive_omm{h[0], h[1], h[2], h[3] ? m_ommIdx[i].data() : nullptr, h[3]};
    }
  }
}

b200pt_scene_desc SceneData::desc() const
{
  b200pt_scene_desc d{};
  d.renderNodes = m_nodes.data();
  d.numRenderNodes = (uint32_t)m_nodes.size();
  d.renderNodeVisible = m_visible.data();
  d.renderPrimitives = m_prims.data();
  d.numRenderPrimitives = (uint32_t)m_prims.size();
  d.materials = m_materials.data();
  d.numMaterials = (uint32_t)m_materials.size();
  d.textureInfos = m_texInfos.data();
  d.numTextureInfos = (uint32_t)m_texInfos.size();
  d.textures = m_textures.data();
  d.numTextures = (uint32_t)m_textures.size();
  d.lights = m_lights.data();
  d.numLights = (uint32_t)m_lights.size();
  return d;
}

size_t SceneData::triangleCount() const
{
  size_t n = 0;
  for(const auto& node : m_nodes)
    n += m_prims[(size_t)node.renderPrimID].triangleCount;
  return n;
}

// ------------------------------------------------------------------------------------------------
// camera math: glm::lookAt / glm::perspectiveRH_ZO with the Vulkan Y flip, in double, rounded once
// ------------------------------------------------------------------------------------------------
namespace {

struct M4
{
  double m[4][4];  // m[row][col]
};

M4 identity()
{
  M4 r{};
  for(int i = 0; i < 4; i++)
    r.m[i][i] = 1.0;
  return r;
}

M4 mul(const M4& a, const M4& b)
{
  M4 r{};
  for(int i = 0; i < 4; i++)
    for(int j = 0; j < 4; j++)
    {
      double s = 0.0;
      for(int k = 0; k < 4; k++)
        s += a.m[i][k] * b.m[k][j];
      r.m[i][j] = s;
    }
  return r;
}

M4 inverse(const M4& a)
{
  // Gauss-Jordan with partial pivoting
  double w[4][8];
  for(int i = 0; i < 4; i++)
    for(int j = 0; j < 4; j++)
    {
      w[i][j] = a.m[i][j];
      w[i][4 + j] = (i == j) ? 1.0 : 0.0;
    }
  for(int c = 0; c < 4; c++)
  {
    int p = c;
    for(int r = c + 1; r < 4; r++)
      if(std::fabs(w[r][c]) > std::fabs(w[p][c]))
        p = r;
    if(w[p][c] == 0.0)
      throw Error("singular camera matrix");
    if(p != c)
      for(int j = 0; j < 8; j++)
        std::swap(w[p][j], w[c][j]);
    const double inv = 1.0 / w[c][c];
    for(int j = 0; j < 8; j++)
      w[c][j] *= inv;
    for(int r = 0; r < 4; r++)
      if(r != c)
      {
        const double f = w[r][c];
        if(f != 0.0)
          for(int j = 0; j < 8; j++)
            w[r][j] -= f * w[c][j];
      }
  }
  M4 r{};
  for(int i = 0; i < 4; i++)
    for(int j = 0; j < 4; j++)
      r.m[i][j] = w[i][4 + j];
  return r;
}

void toGlm(const M4& a, float* out)  // column-major float[16]
{
  for(int c = 0; c < 4; c++)
    for(int r = 0; r < 4; r++)
      out[c * 4 + r] = (float)a.m[r][c];
}

void norm3(double* v)
{
  const double l = std::sqrt(v[0] * v[0] + v[1] * v[1] + v[2] * v[2]);
  v[0] /= l;
  v[1] /= l;
  v[2] /= l;
}

M4 lookAt(const Camera& c)
{
  double f[3] = {(double)c.center[0] - c.eye[0], (double)c.center[1] - c.eye[1], (double)c.center[2] - c.eye[2]};
  norm3(f);
  const double up[3] = {c.up[0], c.up[1], c.up[2]};
  double       s[3] = {f[1] * up[2] - f[2] * up[1], f[2] * up[0] - f[0] * up[2], f[0] * up[1] - f[1] * up[0]};
  norm3(s);
  const double u[3] = {s[1] * f[2] - s[2] * f[1], s[2] * f[0] - s[0] * f[2], s[0] * f[1] - s[1] * f[0]};
  const double e[3] = {c.eye[0], c.eye[1], c.eye[2]};
  M4           m = identity();
  for(int j = 0; j < 3; j++)
  {
    m.m[0][j] = s[j];
    m.m[1][j] = u[j];
    m.m[2][j] = -f[j];
  }
  m.m[0][3] = -(s[0] * e[0] + s[1] * e[1] + s[2] * e[2]);
  m.m[1][3] = -(u[0] * e[0] + u[1] * e[1] + u[2] * e[2]);
  m.m[2][3] = f[0] * e[0] + f[1] * e[1] + f[2] * e[2];
  return m;
}

M4 projection(const Camera& c, double aspect)
{
  M4 m{};
  if(c.orthographic)
  {
    m = identity();
    m.m[0][0] = 1.0 / c.xmag;
    m.m[1][1] = -1.0 / c.ymag;
    m.m[2][2] = -1.0 / ((double)c.zfar - c.znear);
    m.m[2][3] = -(double)c.znear / ((double)c.zfar - c.znear);
    return m;
  }
  const double t = std::tan((double)c.yfov / 2.0);
  m.m[0][0] = 1.0 / (aspect * t);
  m.m[1][1] = -1.0 / t;  // Vulkan clip space: +Y down
  m.m[2][2] = (double)c.zfar / ((double)c.znear - c.zfar);
  m.m[3][2] = -1.0;
  m.m[2][3] = -((double)c.zfar * c.znear) / ((double)c.zfar - c.znear);
  return m;
}

}  // namespace

b200pt_frame_info makeFrameInfo(const Camera& cam, int width, int height, const Settings& s)
{
  const M4          view = lookAt(cam), proj = projection(cam, (double)width / (double)height), vp = mul(proj, view);
  b200pt_frame_info fi{};
  toGlm(view, fi.viewMatrix);
  toGlm(inverse(proj), fi.projInv);
  toGlm(inverse(view), fi.viewInv);
  toGlm(vp, fi.viewProjMatrix);
  toGlm(vp, fi.prevMVP);
  fi.imageSize[0] = (float)width;
  fi.imageSize[1] = (float)height;
  fi.flags = (cam.orthographic ? B200PT_SCENE_IS_ORTHOGRAPHIC : 0) | (s.useSolidBackground ? B200PT_SCENE_USE_SOLID_BACKGROUND : 0)
             | (s.envSystem == 1 ? B200PT_SCENE_USE_HDR_ENVIRONMENT : 0) | (s.useInfinitePlane ? B200PT_SCENE_USE_INFINITE_PLANE : 0)
             | ((s.useInfinitePlane && s.isShadowCatcher) ? B200PT_SCENE_INFINITE_PLANE_SHADOW_CATCHER : 0);  // src/renderer.cpp:688-690
  fi.envRotation = s.hdrEnvRotation;
  fi.envBlur = s.hdrBlur;
  fi.envIntensity = s.hdrEnvIntensity;
  std::memcpy(fi.backgroundColor, s.solidBackgroundColor, 12);
  fi.infinitePlaneDistance = s.infinitePlaneDistance;
  std::memcpy(fi.infinitePlaneBaseColor, s.infinitePlaneBaseColor, 12);
  fi.infinitePlaneMetallic = s.infinitePlaneMetallic;
  fi.infinitePlaneRoughness = s.infinitePlaneRoughness;
  fi.shadowCatcherDarkenAmount = std::max(s.shadowCatcherDarkness, 0.0f);  // src/renderer.cpp:700
  return fi;
}

b200pt_push_constant makePushConstant(const Camera& cam, int height, int frameCount, int totalSamples, const PathTracer& pt)
{
  b200pt_push_constant pc{};
  pc.maxDepth = pt.ptMaxDepth;
  pc.frameCount = frameCount;
  pc.fireflyClampThreshold = pt.ptFireflyClamp;
  pc.texGradScale = pt.ptTexGradScale;
  pc.numSamples = pt.ptSamples;
  pc.totalSamples = totalSamples;
  if(pt.ptAutoFocus)  // focal distance = |eye - center| (renderer_pathtracer.cpp:1508-1512)
  {
    const double d[3] = {(double)cam.eye[0] - cam.center[0], (double)cam.eye[1] - cam.center[1], (double)cam.eye[2] - cam.center[2]};
    pc.focalDistance = (float)std::sqrt(d[0] * d[0] + d[1] * d[1] + d[2] * d[2]);
  }
  else
    pc.focalDistance = pt.ptFocalDistance;
  pc.aperture = pt.ptAperture;
  pc.flags = (frameCount == 0) ? B200PT_PT_FIRST_FRAME : 0;  // ePtFirstFrame (:1542)
  const double projInv11 = cam.orthographic ? (double)cam.ymag : std::tan((double)cam.yfov / 2.0);
  pc.pixelAngle = (float)(2.0 * std::fabs(projInv11) / std::fmax((double)height, 1.0));  // (:1570-1571)
  pc.mouseCoord[0] = pc.mouseCoord[1] = -1.0f;
  return pc;
}

// ------------------------------------------------------------------------------------------------
// PathTracer
// ------------------------------------------------------------------------------------------------
PathTracer::~PathTracer()
{
  if(m_h)
    b200pt_destroy(m_h);
}

void PathTracer::check(int rc, const char* what)
{
  if(rc != B200PT_OK)
    throw Error(std::string(what) + " failed (" + std::to_string(rc) + "): " + (m_h ? b200pt_last_error(m_h) : "no handle"));
}

void PathTracer::onAttach(Resources& res)
{
  const int rc = b200pt_create(&m_h, res.cudaDevice);
  if(rc != B200PT_OK)
    throw Error("b200pt_create failed (" + std::to_string(rc) + "): no usable CUDA device " + std::to_string(res.cudaDevice));
  if(b200pt_abi_version() != B200PT_ABI_VERSION)
    throw Error("libb200pt.so ABI version mismatch");
  if(res.scene)
    onSceneInvalidated(res);
  if(res.hdrRgb)
    check(b200pt_set_environment(m_h, res.hdrRgb, res.hdrWidth, res.hdrHeight, &hdrIntegral), "b200pt_set_environment");
  onResize(res.width, res.height, res);
}

void PathTracer::onDetach(Resources&)
{
  if(m_h)
    b200pt_destroy(m_h);
  m_h = nullptr;
}

void PathTracer::onSceneInvalidated(Resources& res)
{
  const b200pt_scene_desc d = res.scene->desc();
  // SceneOmm::create precedes the BLAS build; --useOpacityMicromap 0 skips the subsystem (src/main.cpp:114-115,349)
  const bool omm = res.settings.useOpacityMicromap && !res.scene->primitiveOmms().empty();
  check(b200pt_set_opacity_micromaps(m_h, res.scene->micromaps().data(), omm ? (uint32_t)res.scene->micromaps().size() : 0u,
                                     res.scene->primitiveOmms().data(), omm ? (uint32_t)res.scene->primitiveOmms().size() : 0u),
        "b200pt_set_opacity_micromaps");
  check(b200pt_set_scene(m_h, &d), "b200pt_set_scene");
}

void PathTracer::onResize(int width, int height, Resources& res)
{
  if(res.bandWorld > 1)
  {
    check(b200pt_resize_interleaved(m_h, width, height, res.bandRows, res.bandWorld, res.bandRank), "b200pt_resize_interleaved");
    m_tileRows = height / res.bandWorld;
  }
  else
  {
    m_tileRows = res.tileRows > 0 ? res.tileRows : height;
    check(b200pt_resize(m_h, width, height, res.tileRows > 0 ? res.tileY0 : 0, m_tileRows), "b200pt_resize");
  }
  m_width = width;
  m_height = height;
  res.width = width;
  res.height = height;
}

void PathTracer::updateAdaptiveSampling(const Resources& res)
{
  constexpr int kMin = 1, kMax = 100;  // MIN_/MAX_SAMPLES_PER_PIXEL
  if(!ptAdaptiveSampling)
    return;
  if(res.frameCount == 0)
  {
    ptSamples = kMin;  // the accumulation restarted
    return;
  }
  if(res.frameCount < 5 || lastFrameGpuMs < 0.0)
    return;
  static const double kTarget[4] = {1000.0 / 60.0, 1000.0 / 30.0, 1000.0 / 15.0, 1000.0 / 10.0};
  const double        target = kTarget[std::min(std::max(ptPerformanceTarget, 0), 3)];
  if(lastFrameGpuMs < target * 0.8 && ptSamples < kMax)
    ptSamples++;
  else if(lastFrameGpuMs > target * 1.1 && ptSamples > kMin)
    ptSamples--;
  ptSamples = std::min(std::max(ptSamples, kMin), kMax);
}

void PathTracer::onRender(Resources& res)
{
  updateAdaptiveSampling(res);
  if(res.frameCount == 0)
    m_totalSamplesAccumulated = 0;
  const b200pt_frame_info fi = makeFrameInfo(res.camera, m_width, m_height, res.settings);
  m_pushConst = makePushConstant(res.camera, m_height, res.frameCount, m_totalSamplesAccumulated, *this);
  check(b200pt_render_frame(m_h, &fi, &m_pushConst), "b200pt_render_frame");
  m_totalSamplesAccumulated += ptSamples;  // updateStatistics (renderer_pathtracer.cpp:1377-1402)
}

void PathTracer::registerParameters(std::map<std::string, std::string>& registry)
{
  registry["ptMaxDepth"] = std::to_string(ptMaxDepth);
  registry["ptSamples"] = std::to_string(ptSamples);
  registry["ptFireflyClamp"] = std::to_string(ptFireflyClamp);
  registry["ptTexGradScale"] = std::to_string(ptTexGradScale);
  registry["ptAperture"] = std::to_string(ptAperture);
  registry["ptFocalDistance"] = std::to_string(ptFocalDistance);
  registry["ptAutoFocus"] = ptAutoFocus ? "1" : "0";
  registry["ptAdaptiveSampling"] = ptAdaptiveSampling ? "1" : "0";
  registry["ptPerformanceTarget"] = std::to_string(ptPerformanceTarget);
}

bool PathTracer::setParameter(const std::string& name, const std::string& value)
{
  if(name == "ptMaxDepth")
    ptMaxDepth = std::stoi(value);
  else if(name == "ptSamples")
    ptSamples = std::stoi(value);
  else if(name == "ptFireflyClamp")
    ptFireflyClamp = std::stof(value);
  else if(name == "ptTexGradScale")
    ptTexGradScale = std::stof(value);
  else if(name == "ptAperture")
    ptAperture = std::stof(value);
  else if(name == "ptFocalDistance")
    ptFocalDistance = std::stof(value);
  else if(name == "ptAutoFocus")
    ptAutoFocus = std::stoi(value) != 0;
  else if(name == "ptAdaptiveSampling")
    ptAdaptiveSampling = std::stoi(value) != 0;
  else if(name == "ptPerformanceTarget")
    ptPerformanceTarget = std::stoi(value);
  else
    return false;
  return true;
}

std::vector<float> PathTracer::readAccum()
{
  std::vector<float> img((size_t)m_width * (size_t)m_tileRows * 4);
  check(b200pt_read_accum(m_h, img.data(), img.size()), "b200pt_read_accum");
  return img;
}

std::vector<uint8_t> PathTracer::tonemap(const b200pt_tonemapper& tm, float* exposureUsed)
{
  std::vector<uint8_t> img((size_t)m_width * (size_t)m_tileRows * 4);
  check(b200pt_tonemap(m_h, &tm, img.data(), img.size(), exposureUsed), "b200pt_tonemap");
  return img;
}

void PathTracer::setAnimation(const std::vector<b200pt_morph_task>& morphs, const std::vector<b200pt_skin_task>& skins)
{
  check(b200pt_set_animation(m_h, morphs.data(), (uint32_t)morphs.size(), skins.data(), (uint32_t)skins.size()), "b200pt_set_animation");
}

void PathTracer::animate(const std::vector<float>& morphWeights, const std::vector<float>& jointMatrices, const std::vector<float>& normalMatrices)
{
  check(b200pt_animate(m_h, morphWeights.data(), jointMatrices.data(), normalMatrices.data()), "b200pt_animate");
}

void PathTracer::synchronize() { check(b200pt_synchronize(m_h), "b200pt_synchronize"); }

void PathTracer::setFramesInFlight(int n) { check(b200pt_set_frames_in_flight(m_h, n), "b200pt_set_frames_in_flight"); }

void PathTracer::setFrameBatch(int n) { check(b200pt_set_frame_batch(m_h, n), "b200pt_set_frame_batch"); }

void PathTracer::flush() { check(b200pt_flush(m_h), "b200pt_flush"); }

void PathTracer::setViews(int n) { check(b200pt_set_views(m_h, n), "b200pt_set_views"); }

void PathTracer::renderViews(const std::vector<b200pt_frame_info>& fis, const b200pt_push_constant& pc)
{
  check(b200pt_render_views(m_h, fis.data(), (uint32_t)fis.size(), &pc), "b200pt_render_views");
}

std::vector<float> PathTracer::readView(uint32_t view, std::vector<uint32_t>* objectIds, std::vector<float>* ndcDepth)
{
  const size_t       n = (size_t)m_width * m_tileRows;
  std::vector<float> rgba(n * 4);
  if(objectIds)
    objectIds->resize(n);
  if(ndcDepth)
    ndcDepth->resize(n);
  check(b200pt_read_views(m_h, view, rgba.data(), objectIds ? objectIds->data() : nullptr, ndcDepth ? ndcDepth->data() : nullptr, n), "b200pt_read_views");
  return rgba;
}

b200pt_stats PathTracer::stats()
{
  b200pt_stats s{};
  check(b200pt_get_stats(m_h, &s), "b200pt_get_stats");
  return s;
}

void PathTracer::resetStats() { check(b200pt_reset_stats(m_h), "b200pt_reset_stats"); }

std::vector<float> renderHeadless(PathTracer& pt, Resources& res, int frames)
{
  res.frameCount = -1;
  for(int f = 0; f < frames; f++)
  {
    res.frameCount++;
    pt.onRender(res);
  }
  return pt.readAccum();
}

}  // namespace b200host
