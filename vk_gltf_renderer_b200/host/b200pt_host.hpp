// b200pt_host.hpp — C++ host side above the C-ABI (include/b200pt.h).
//
// The reference's path tracer sits behind the C++ virtual class BaseRenderer (reference src/renderer_base.hpp:33-55)
// and is driven by GltfRenderer with a `Resources` bag (src/resources.hpp:167-276).  This header mirrors that
// interface — same method names, parameter names (`--pt*`, src/renderer_pathtracer.cpp:119-132) and error behaviour
// (a failed call is fatal: NVVK_CHECK aborts there, an exception carrying b200pt_last_error() here) — so that the
// class below is what a maintainer would drop into the reference in place of `PathTracer` (see INTEGRATION.md).
// Standalone it is driven by host/headless_main.cpp, the stand-in for `vk_gltf_renderer --headless`.
//
// There is no CPU rendering path in here: every virtual is a call into libb200pt.so.
#pragma once
#include <cstdint>
#include <map>
#include <stdexcept>
#include <string>
#include <vector>

#include "b200pt.h"

namespace b200host {

struct Error : std::runtime_error
{
  using std::runtime_error::runtime_error;
};

// Resources::settings (reference src/resources.hpp:82-133): the fields the path tracer reads
struct Settings
{
  int   envSystem           = 1;  // 0 sky (not built: the frame call fails), 1 HDR
  float hdrEnvIntensity     = 1.0f;
  float hdrEnvRotation      = 0.0f;
  float hdrBlur             = 0.0f;
  bool  useSolidBackground  = false;
  float solidBackgroundColor[3] = {0.f, 0.f, 0.f};
  int   maxFrames           = 500;
  // infinite ground plane (src/resources.hpp:111-117); like the reference it is a shadow catcher unless told otherwise
  bool  useInfinitePlane       = false;
  bool  isShadowCatcher        = true;
  float infinitePlaneDistance  = 0.0f;
  float infinitePlaneBaseColor[3] = {0.5f, 0.5f, 0.5f};
  float infinitePlaneMetallic  = 0.0f;
  float infinitePlaneRoughness = 0.5f;
  float shadowCatcherDarkness  = 0.0f;
  bool  useOpacityMicromap     = true;  // --useOpacityMicromap (src/main.cpp:114-115): consume EXT_mesh_opacity_micromap when the asset has it
};

// what nvutils::CameraManipulator hands the renderer (external to the reference tree): look-at + lens
struct Camera
{
  bool  orthographic = false;
  float eye[3] = {0, 0, 1}, center[3] = {0, 0, 0}, up[3] = {0, 1, 0};
  float yfov = 0.785398f, znear = 0.1f, zfar = 1000.f, xmag = 1.f, ymag = 1.f;
};

// The arrays SceneVk / MaterialCache / SceneRtx upload in the reference (src/gltf_scene_vk.cpp:218-252), owned on the
// host.  load() reads the "B2SC" blob written by vk_gltf_renderer_b200.scene.Scene.save_blob().
class SceneData
{
public:
  void load(const std::string& path);  // throws Error
  b200pt_scene_desc desc() const;      // pointers into this object
  Camera             camera;
  std::vector<float> hdrRgb;           // optional environment carried by the blob
  int                hdrWidth = 0, hdrHeight = 0;
  size_t             triangleCount() const;
  // EXT_mesh_opacity_micromap arrays carried by the blob (empty when the asset has none)
  const std::vector<b200pt_micromap>&      micromaps() const { return m_micromaps; }
  const std::vector<b200pt_primitive_omm>& primitiveOmms() const { return m_primOmms; }

private:
  struct Prim
  {
    std::vector<float>    positions, normals, uv0, uv1, tangents;
    std::vector<uint32_t> indices, colors;
  };
  std::vector<b200pt_render_node>      m_nodes;
  std::vector<uint8_t>                 m_visible;
  std::vector<Prim>                    m_primData;
  std::vector<b200pt_render_primitive> m_prims;
  std::vector<b200pt_shade_material>   m_materials;
  std::vector<b200pt_texture_info>     m_texInfos;
  std::vector<std::vector<uint8_t>>    m_texPixels;
  std::vector<b200pt_texture>          m_textures;
  std::vector<b200pt_light>            m_lights;
  std::vector<std::vector<uint8_t>>                  m_ommData;
  std::vector<std::vector<b200pt_micromap_triangle>> m_ommTris;
  std::vector<std::vector<int32_t>>                  m_ommIdx;
  std::vector<b200pt_micromap>                       m_micromaps;
  std::vector<b200pt_primitive_omm>                  m_primOmms;
};

// the subset of the reference's Resources the path tracer touches
struct Resources
{
  const SceneData* scene = nullptr;
  const float*     hdrRgb = nullptr;  // float3 per texel, row 0 first
  int              hdrWidth = 0, hdrHeight = 0;
  Camera           camera;
  Settings         settings;
  // Resources::tonemapperData (src/resources.hpp:212: the reference turns auto-exposure on): filmic, neutral controls
  b200pt_tonemapper tonemapperData{0, 1, 1.0f, 1.0f, 1.0f, 1.0f, 0.0f, 1};
  int              width = 1920, height = 1080;
  int              frameCount = -1;  // reset to -1 and pre-incremented by the frame loop (src/renderer.cpp:1939-1977)
  int              cudaDevice = 0;
  // multi-GPU tile: tileRows == 0 -> whole image; bandWorld > 1 -> interleaved bands
  int tileY0 = 0, tileRows = 0, bandRows = 0, bandWorld = 1, bandRank = 0;
};

// reference src/renderer_base.hpp:33-55
class BaseRenderer
{
public:
  virtual ~BaseRenderer() = default;
  virtual void onAttach(Resources& res)                           = 0;
  virtual void onDetach(Resources& res)                           = 0;
  virtual void onResize(int width, int height, Resources& res)    = 0;
  virtual void onRender(Resources& res)                           = 0;
  virtual void onSceneInvalidated(Resources& res)                 = 0;
  virtual bool onUIRender(Resources&) { return false; }           // no UI on this side of the boundary
  virtual void registerParameters(std::map<std::string, std::string>& registry) = 0;
};

// reference src/renderer_pathtracer.hpp:61-88
class PathTracer : public BaseRenderer
{
public:
  PathTracer() = default;
  ~PathTracer() override;
  PathTracer(const PathTracer&)            = delete;
  PathTracer& operator=(const PathTracer&) = delete;

  void onAttach(Resources& res) override;
  void onDetach(Resources& res) override;
  void onResize(int width, int height, Resources& res) override;
  void onRender(Resources& res) override;
  void onSceneInvalidated(Resources& res) override;
  void registerParameters(std::map<std::string, std::string>& registry) override;
  bool setParameter(const std::string& name, const std::string& value);  // "--ptMaxDepth 12" style

  // --pt* parameters (src/renderer_pathtracer.cpp:119-132), defaults of PathtracePushConstant (shaders/shaderio.h:181-190)
  int   ptMaxDepth      = 5;
  int   ptSamples       = 1;
  float ptFireflyClamp  = 10.0f;
  float ptTexGradScale  = 1.0f;
  float ptAperture      = 0.0f;
  float ptFocalDistance = 0.0f;
  bool  ptAutoFocus     = true;
  // adaptive sampling (reference src/renderer_pathtracer.hpp:158-199): OFF by default here (the harness passes 0)
  bool   ptAdaptiveSampling  = false;
  int    ptPerformanceTarget = 1;      // 0: 60 FPS, 1: 30, 2: 15, 3: 10
  double lastFrameGpuMs      = -1.0;   // GPU time of the previous frame's path-trace section, < 0 = unknown
  void   updateAdaptiveSampling(const Resources& res);  // src/renderer_pathtracer.cpp:1326-1374

  b200pt_push_constant m_pushConst{};
  int                  m_totalSamplesAccumulated = 0;
  float                hdrIntegral               = 0.f;

  // gBuffers[eImgRendered] (RGBA32F running mean) of this renderer's tile
  std::vector<float> readAccum();
  // GltfRenderer::tonemap (src/renderer.cpp:992-1054): gBuffers[eImgRendered] -> gBuffers[eImgTonemapped] (RGBA8) of this tile
  std::vector<uint8_t> tonemap(const b200pt_tonemapper& tm, float* exposureUsed = nullptr);
  // SceneAnimationVk::createAnimationResources / cmdUpdateAnimation analogues (b200pt_set_animation / b200pt_animate)
  void setAnimation(const std::vector<b200pt_morph_task>& morphs, const std::vector<b200pt_skin_task>& skins);
  void animate(const std::vector<float>& morphWeights, const std::vector<float>& jointMatrices, const std::vector<float>& normalMatrices);
  void               synchronize();
  void               setFramesInFlight(int n);
  void               setFrameBatch(int n);  // b200pt_set_frame_batch
  void               flush();               // b200pt_flush
  // views (b200pt_set_views / b200pt_render_views): n poses of one frame as one wavefront, each into its own images; readView(v) is
  // view v's RGBA32F image of this tile, with its object ids and NDC depth when asked for
  void               setViews(int n);
  void               renderViews(const std::vector<b200pt_frame_info>& fis, const b200pt_push_constant& pc);
  std::vector<float> readView(uint32_t view, std::vector<uint32_t>* objectIds = nullptr, std::vector<float>* ndcDepth = nullptr);
  b200pt_stats       stats();
  void               resetStats();
  b200pt_t*          handle() { return m_h; }
  int                tileRows() const { return m_tileRows; }

private:
  void      check(int rc, const char* what);
  b200pt_t* m_h = nullptr;
  int       m_width = 0, m_height = 0, m_tileRows = 0;
};

// SceneFrameInfo as GltfRenderer::onRender fills it every frame (src/renderer.cpp:677-700) and the pointer-less part of
// PathtracePushConstant as PathTracer::setupPushConstant does (src/renderer_pathtracer.cpp:1496-1574)
b200pt_frame_info    makeFrameInfo(const Camera& cam, int width, int height, const Settings& s);
b200pt_push_constant makePushConstant(const Camera& cam, int height, int frameCount, int totalSamples, const PathTracer& pt);

// the reference's headless frame loop (src/main.cpp:133-136 + nvapp): frames x onRender, returns the accumulation image
std::vector<float> renderHeadless(PathTracer& pt, Resources& res, int frames);

}  // namespace b200host
