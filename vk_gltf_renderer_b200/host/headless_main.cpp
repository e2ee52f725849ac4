// headless_main.cpp — stand-in for `vk_gltf_renderer --headless --frames N --ptSamples S …` (reference src/main.cpp:133-136,
// headless flow src/renderer.cpp:1939-1977, summary lines src/benchmarking.cpp:245-305) on top of the C++ host mirror.
//
// Accepts the command line the reference's benchmark harness spawns (utils/benchmark/benchmark_runner.py:164-198):
//   b200pt_headless --headless --size W H --frames N --maxFrames N --ptSamples S --ptAdaptiveSampling 0 --renderSystem 0
//                   --envSystem 1 --scenefile scene.glb [--hdrfile env.hdr] [extra args]
// plus  --scene scene.b2sc  (a pre-converted blob), --warmupFrames K, --device G, --framesInFlight L, --out image.pfm,
// --outRaw image.f32, and the library's own convergence flags (not the reference's): --ptConvergenceThreshold T (0 = off),
// --ptConvergenceMinFrames M (16) and --ptConvergenceInterval I (8).  With a threshold the run ends at --frames or after the first
// checkpoint at which no pixel is still active, whichever comes first (include/b200pt.h, b200pt_set_convergence).  A .gltf / .glb scene is converted on the fly by the package's own loader
// (python -m vk_gltf_renderer_b200.convert).  Flags of the reference application that have no meaning for this backend are
// skipped with a note on stderr; --renderSystem other than 0 (path tracer) and --envSystem 0 (physical sky) are errors.
//
// Prints the reference's record kinds so its benchmark tooling reads them unchanged (utils/benchmark/benchmark_results.py):
// "HEADLESS_PROGRESS …" / "HEADLESS_SUMMARY key=value …" lines and "BENCHMARK_JSON {"schema":1, …}" records with the same
// keys, plus the ray counters the reference lacks.  Like the reference, the first frame is warm-up and excluded from the
// measured window (kHeadlessWarmupFrames = 1, src/benchmarking.hpp:128), and maxFrames is raised to the number of frames
// (alignMaxFramesForHeadless).  The image written by --out is the RGBA32F accumulation buffer (what the reference tonemaps).
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <unistd.h>

#include "b200pt_host.hpp"
#include "b2sc_writer.hpp"

using namespace b200host;

static void writePfm(const std::string& path, const std::vector<float>& rgba, int w, int h)
{
  FILE* f = std::fopen(path.c_str(), "wb");
  if(!f)
    throw Error("cannot write " + path);
  std::fprintf(f, "PF\n%d %d\n-1.0\n", w, h);
  std::vector<float> row((size_t)w * 3);
  for(int y = h - 1; y >= 0; y--)  // PFM stores the bottom row first
  {
    for(int x = 0; x < w; x++)
      for(int c = 0; c < 3; c++)
        row[(size_t)x * 3 + c] = rgba[((size_t)y * w + x) * 4 + c];
    std::fwrite(row.data(), sizeof(float), row.size(), f);
  }
  std::fclose(f);
}

static void writePpm(const std::string& path, const std::vector<uint8_t>& rgba, int w, int h)
{
  FILE* f = std::fopen(path.c_str(), "wb");
  if(!f)
    throw Error("cannot write " + path);
  std::fprintf(f, "P6\n%d %d\n255\n", w, h);
  std::vector<uint8_t> row((size_t)w * 3);
  for(int y = 0; y < h; y++)
  {
    for(int x = 0; x < w; x++)
      for(int c = 0; c < 3; c++)
        row[(size_t)x * 3 + c] = rgba[((size_t)y * w + x) * 4 + c];
    std::fwrite(row.data(), 1, row.size(), f);
  }
  std::fclose(f);
}

static void writeRaw(const std::string& path, const std::vector<float>& rgba)
{
  FILE* f = std::fopen(path.c_str(), "wb");
  if(!f)
    throw Error("cannot write " + path);
  std::fwrite(rgba.data(), sizeof(float), rgba.size(), f);
  std::fclose(f);
}

static bool endsWith(const std::string& s, const char* suffix)
{
  const size_t n = std::strlen(suffix);
  return s.size() >= n && s.compare(s.size() - n, n, suffix) == 0;
}

// .gltf / .glb (+ .hdr) -> temporary B2SC blob through the package's loader; returns the blob path
static std::string convertScene(const std::string& gltf, const std::string& hdrFile)
{
  char self[4096];
  const ssize_t n = readlink("/proc/self/exe", self, sizeof(self) - 1);
  if(n <= 0)
    throw Error("cannot locate the executable (needed to find the vk_gltf_renderer_b200 package)");
  self[n] = 0;
  std::string pkgDir(self);
  pkgDir = pkgDir.substr(0, pkgDir.find_last_of('/'));                  // .../vk_gltf_renderer_b200
  const std::string root = pkgDir.substr(0, pkgDir.find_last_of('/'));  // repo root (PYTHONPATH)
  char              tmpl[] = "/tmp/b200pt_scene_XXXXXX";
  const int         fd = mkstemp(tmpl);
  if(fd < 0)
    throw Error("cannot create a temporary scene blob");
  close(fd);
  auto quote = [](const std::string& p) {
    std::string q = "'";
    for(char c : p)
      q += (c == '\'') ? std::string("'\\''") : std::string(1, c);
    return q + "'";
  };
  const char*       py = std::getenv("B200PT_PYTHON");
  const std::string cmd = "PYTHONPATH=" + quote(root) + ":\"$PYTHONPATH\" " + std::string(py ? py : "python3") + " -m vk_gltf_renderer_b200.convert " + quote(gltf) + " "
                          + quote(tmpl) + (hdrFile.empty() ? std::string() : " --hdr " + quote(hdrFile)) + " 1>&2";
  if(std::system(cmd.c_str()) != 0)
  {
    unlink(tmpl);
    throw Error("scene conversion failed: " + cmd);
  }
  return tmpl;
}

int main(int argc, char** argv)
{
  std::string scenePath, hdrPath, outPath, rawPath, tmpBlob, tonemappedPath, writeBlobPath;
  int         width = 1920, height = 1080, frames = 16, warmupFrames = 1, framesInFlight = 0;  // warm-up: src/benchmarking.hpp:128
  int         adaptiveSampling = 0, frameBatch = 0;
  b200pt_convergence convergence{0.0f, 1e-3f, 16u, 8u};
  Resources   res;
  PathTracer  pt;
  try
  {
    for(int i = 1; i < argc; i++)
    {
      const std::string a = argv[i];
      auto              next = [&]() -> std::string {
        if(i + 1 >= argc)
          throw Error("missing value after " + a);
        return argv[++i];
      };
      if(a == "--scene" || a == "--scenefile")
        scenePath = next();
      else if(a == "--hdrfile")
        hdrPath = next();
      else if(a == "--headless")
      {
      }
      else if(a == "--renderSystem")
      {
        if(std::stoi(next()) != 0)
          throw Error("--renderSystem: only 0 (path tracer) is this backend's path");
      }
      else if(a == "--ptAdaptiveSampling")
      {
        adaptiveSampling = std::stoi(next());
        pt.ptAdaptiveSampling = adaptiveSampling != 0;
      }
      else if(a == "--size")
      {
        width = std::stoi(next());
        height = std::stoi(next());
      }
      else if(a == "--frames")
        frames = std::stoi(next());
      else if(a == "--warmupFrames")
        warmupFrames = std::stoi(next());
      else if(a == "--device")
        res.cudaDevice = std::stoi(next());
      else if(a == "--framesInFlight")
        framesInFlight = std::stoi(next());
      else if(a == "--frameBatch")
        frameBatch = std::stoi(next());
      else if(a == "--maxFrames")
        res.settings.maxFrames = std::stoi(next());
      else if(a == "--hdrEnvIntensity")
        res.settings.hdrEnvIntensity = std::stof(next());
      else if(a == "--hdrEnvRotation")
        res.settings.hdrEnvRotation = std::stof(next());
      else if(a == "--envSystem")
        res.settings.envSystem = std::stoi(next());
      else if(a == "--useOpacityMicromap")
        res.settings.useOpacityMicromap = std::stoi(next()) != 0;
      else if(a == "--out")
        outPath = next();
      else if(a == "--writeBlob")
        writeBlobPath = next();  // re-serialise the loaded scene with host/b2sc_writer.hpp and exit (no GPU needed: round-trip check)
      else if(a == "--output" || a == "--screenshot")
        tonemappedPath = next();  // the reference's headless output image (src/renderer.cpp:171, 557-573; benchmarking.cpp:144-153)
      else if(a == "--tonemapMethod")
        res.tonemapperData.method = std::stoi(next());
      else if(a == "--tonemapAutoExposure")
        res.tonemapperData.autoExposure = std::stoi(next());
      else if(a == "--tonemapExposure")
        res.tonemapperData.exposure = std::stof(next());
      else if(a == "--outRaw")
        rawPath = next();
      else if(a == "--ptConvergenceThreshold")
        convergence.threshold = std::stof(next());
      else if(a == "--ptConvergenceMinFrames")
        convergence.minFrames = (uint32_t)std::stoul(next());
      else if(a == "--ptConvergenceInterval")
        convergence.interval = (uint32_t)std::stoul(next());
      else if(a.rfind("--pt", 0) == 0)
      {
        if(!pt.setParameter(a.substr(2), next()))
          throw Error("unknown parameter " + a);
      }
      else if(a.rfind("--", 0) == 0)
      {
        // a flag of the reference application without meaning here: skip it and its value(s)
        std::fprintf(stderr, "b200pt_headless: ignoring %s", a.c_str());
        while(i + 1 < argc && std::strncmp(argv[i + 1], "--", 2) != 0)
          std::fprintf(stderr, " %s", argv[++i]);
        std::fprintf(stderr, "\n");
      }
      else
        throw Error("unknown argument " + a);
    }
    (void)adaptiveSampling;  // 0 in every harness run; the controller itself lives in PathTracer::updateAdaptiveSampling
    if(scenePath.empty())
      throw Error("usage: b200pt_headless --scenefile scene.glb|scene.b2sc [--hdrfile env.hdr] [--size W H] [--frames N] [--pt<Name> value] [--out image.pfm]");
    // alignMaxFramesForHeadless (src/benchmarking.hpp:112): accumulation keeps refining for the whole capture
    if(res.settings.maxFrames < frames)
      res.settings.maxFrames = frames;
    warmupFrames = std::min(warmupFrames, std::max(frames - 1, 0));
    if(endsWith(scenePath, ".gltf") || endsWith(scenePath, ".glb"))
    {
      tmpBlob = convertScene(scenePath, hdrPath);
      scenePath = tmpBlob;
    }
    else if(!hdrPath.empty())
      std::fprintf(stderr, "b200pt_headless: --hdrfile is read during glTF conversion only; a .b2sc blob carries its own environment\n");

    SceneData scene;
    scene.load(scenePath);
    if(!tmpBlob.empty())
      unlink(tmpBlob.c_str());
    if(!writeBlobPath.empty())
    {
      BlobCamera bc;
      bc.orthographic = scene.camera.orthographic ? 1u : 0u;
      std::memcpy(bc.eye, scene.camera.eye, 12), std::memcpy(bc.center, scene.camera.center, 12), std::memcpy(bc.up, scene.camera.up, 12);
      bc.yfov = scene.camera.yfov, bc.znear = scene.camera.znear, bc.zfar = scene.camera.zfar, bc.xmag = scene.camera.xmag, bc.ymag = scene.camera.ymag;
      const b200pt_scene_desc d = scene.desc();
      writeB2sc(writeBlobPath, d, bc, scene.hdrRgb.empty() ? nullptr : scene.hdrRgb.data(), (uint32_t)scene.hdrWidth, (uint32_t)scene.hdrHeight,
                scene.micromaps().data(), (uint32_t)scene.micromaps().size(), scene.primitiveOmms().data(), (uint32_t)scene.primitiveOmms().size());
      std::printf("wrote %s\n", writeBlobPath.c_str());
      return 0;
    }
    res.scene = &scene;
    res.camera = scene.camera;
    res.width = width;
    res.height = height;
    if(!scene.hdrRgb.empty())
    {
      res.hdrRgb = scene.hdrRgb.data();
      res.hdrWidth = scene.hdrWidth;
      res.hdrHeight = scene.hdrHeight;
    }
    pt.onAttach(res);
    if(framesInFlight > 0)
      pt.setFramesInFlight(framesInFlight);
    if(frameBatch > 0)
      pt.setFrameBatch(frameBatch);
    const bool converge = convergence.threshold != 0.0f;
    if(converge && b200pt_set_convergence(pt.handle(), &convergence) != B200PT_OK)
      throw Error(std::string("b200pt_set_convergence: ") + b200pt_last_error(pt.handle()));

    // frame loop with the reference's warm-up split (benchmarking.cpp: measured timer starts after warmupFrames)
    using clock = std::chrono::steady_clock;
    const auto t0 = clock::now();
    auto       tMeasured = t0;
    res.frameCount = -1;
    for(int f = 0; f < frames; f++)
    {
      if(f == warmupFrames)
      {
        pt.synchronize();
        pt.resetStats();
        tMeasured = clock::now();
      }
      res.frameCount++;
      pt.onRender(res);
      if(converge && (f + 1) % (int)convergence.interval == 0)
      {
        // the count synchronises, so it is read at checkpoints only: the mask changes nowhere else
        uint32_t active = 0;
        if(b200pt_read_convergence(pt.handle(), nullptr, nullptr, 0, &active) != B200PT_OK)
          throw Error(std::string("b200pt_read_convergence: ") + b200pt_last_error(pt.handle()));
        if(active == 0)
        {
          std::printf("HEADLESS_CONVERGED frame=%d frames=%d: no pixel is active\n", f, f + 1);
          frames = f + 1;
          break;
        }
      }
      if((f + 1) % 50 == 0 && f + 1 < frames)
      {
        // progress records like updateHeadlessProgressIfNeeded (src/benchmarking.cpp:215-238), every 50 frames; the
        // frames are only SUBMITTED at this point (frames in flight), like the reference's app_frame counter
        const double el = std::chrono::duration<double, std::milli>(clock::now() - t0).count();
        std::printf("HEADLESS_PROGRESS app_frame %d/%d (%.0f%%) elapsed_ms=%.1f ms_per_frame=%.2f\n", f + 1, frames, 100.0 * (f + 1) / frames, el, el / (f + 1));
        std::printf("BENCHMARK_JSON {\"schema\":1,\"type\":\"headless_progress\",\"app_frame\":%d,\"frames\":%d,\"percent\":%.3f,\"elapsed_ms\":%.3f,\"ms_per_frame\":%.3f}\n",
                    f + 1, frames, 100.0 * (f + 1) / frames, el, el / (f + 1));
      }
    }
    pt.synchronize();
    const auto   t1 = clock::now();
    const double totalWallMs = std::chrono::duration<double, std::milli>(t1 - t0).count();
    const double measuredWallMs = std::chrono::duration<double, std::milli>(t1 - tMeasured).count();
    const int    measuredFrames = frames - warmupFrames;
    const int    accumFrames = std::min(frames, std::max(res.settings.maxFrames, 0));
    const int    effectiveSpp = accumFrames * std::max(pt.ptSamples, 1);
    const int    measuredEffectiveSpp = std::max(0, std::min(accumFrames - warmupFrames, measuredFrames)) * std::max(pt.ptSamples, 1);
    const double sec = measuredWallMs / 1000.0;
    const double throughputMSps = sec > 0 ? (double)width * height * measuredEffectiveSpp / sec / 1e6 : 0.0;
    const double sppPerSec = sec > 0 ? measuredEffectiveSpp / sec : 0.0;
    const b200pt_stats st = pt.stats();
    const double       mrays = sec > 0 ? (double)(st.closestRays + st.shadowRays) / sec / 1e6 : 0.0;

    std::printf(
        "HEADLESS_SUMMARY frames=%d maxFrames=%d ptSamples=%d effective_spp=%d measured_effective_spp=%d resolution=%dx%d wall_ms=%.3f "
        "ms_per_frame=%.3f total_wall_ms=%.3f total_ms_per_frame=%.3f warmup_frames=%d measured_frames=%d throughput_MSps=%.3f spp_per_sec=%.2f\n",
        frames, res.settings.maxFrames, pt.ptSamples, effectiveSpp, measuredEffectiveSpp, width, height, measuredWallMs,
        measuredFrames > 0 ? measuredWallMs / measuredFrames : 0.0, totalWallMs, frames > 0 ? totalWallMs / frames : 0.0, warmupFrames, measuredFrames,
        throughputMSps, sppPerSec);
    std::printf(
        "BENCHMARK_JSON {\"schema\":1,\"type\":\"headless_summary\",\"frames\":%d,\"maxFrames\":%d,\"ptSamples\":%d,\"effective_spp\":%d,"
        "\"measured_effective_spp\":%d,\"resolution_w\":%d,\"resolution_h\":%d,\"wall_ms\":%.3f,\"ms_per_frame\":%.3f,\"total_wall_ms\":%.3f,"
        "\"total_ms_per_frame\":%.3f,\"warmup_frames\":%d,\"measured_frames\":%d,\"throughput_MSps\":%.3f,\"spp_per_sec\":%.2f,"
        "\"closest_rays\":%llu,\"shadow_rays\":%llu,\"Mray_per_s\":%.3f,\"triangles\":%zu,\"backend\":\"b200pt\"}\n",
        frames, res.settings.maxFrames, pt.ptSamples, effectiveSpp, measuredEffectiveSpp, width, height, measuredWallMs,
        measuredFrames > 0 ? measuredWallMs / measuredFrames : 0.0, totalWallMs, frames > 0 ? totalWallMs / frames : 0.0, warmupFrames, measuredFrames,
        throughputMSps, sppPerSec, (unsigned long long)st.closestRays, (unsigned long long)st.shadowRays, mrays, scene.triangleCount());

    if(!tonemappedPath.empty())
    {
      // saveHeadlessOutputImage: the tonemapped 8-bit image.  The reference encodes .jpg / .png through its image library; this
      // driver has no encoder and writes the same pixels as a binary PPM (P6, alpha dropped), whatever the extension says.
      float                      ex = 1.0f;
      const std::vector<uint8_t> rgba = pt.tonemap(res.tonemapperData, &ex);
      writePpm(tonemappedPath, rgba, width, pt.tileRows());
      std::printf("HEADLESS_OUTPUT path=%s format=ppm tonemap_method=%d auto_exposure=%d exposure=%.6g\n", tonemappedPath.c_str(), res.tonemapperData.method,
                  res.tonemapperData.autoExposure, ex);
    }
    if(!outPath.empty() || !rawPath.empty())
    {
      const std::vector<float> img = pt.readAccum();
      if(!outPath.empty())
        writePfm(outPath, img, width, pt.tileRows());
      if(!rawPath.empty())
        writeRaw(rawPath, img);
    }
    pt.onDetach(res);
  }
  catch(const std::exception& e)
  {
    std::fprintf(stderr, "b200pt_headless: %s\n", e.what());
    return 1;
  }
  return 0;
}
