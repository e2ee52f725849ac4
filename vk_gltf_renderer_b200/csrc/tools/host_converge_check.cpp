// host_converge_check.cpp — the convergence rule (converge.cuh: convergeLum / convergeUpdate / convergeRelError / convergeStops, what
// k_accumulate<true> runs) compiled for the host and driven by a synthetic frame stream from tests/test_convergence.py.  The image fold
// restates k_accumulate's running mean op for op, so M2, e and the stop frames are those the device computes for the same pixel sums.
//   host_converge_check in.bin out.bin
// in.bin:  u32 pixels, frames; the rule (f32 threshold, floor, u32 minFrames, interval); per frame i32 numSamples, then RGBA32F pixel
//          sums (the frame's clamped samples summed in order, P.pixSum).
// out.bin: u32 stop frame per pixel; then per frame f32 M2 per pixel and f32 e per pixel (NaN for a pixel stopped before the frame).
#include "host_shim.h"

#include <cstdio>
#include <vector>

#include "../converge.cuh"

using namespace pt;

int main(int argc, char** argv)
{
  if(argc < 3)
    return 2;
  FILE* f = std::fopen(argv[1], "rb");
  if(!f)
    return 2;
  uint32_t     hd[2];
  ConvergeRule rule;
  if(std::fread(hd, 4, 2, f) != 2 || std::fread(&rule, sizeof(rule), 1, f) != 1)
    return 2;
  const uint32_t        n = hd[0], frames = hd[1];
  std::vector<float4>   sum(n), img(n);
  std::vector<float>    m2(n, 0.0f), outM2(n), outE(n);
  std::vector<uint32_t> stop(n, 0u);
  FILE*                 o = std::fopen(argv[2], "wb");
  if(!o)
    return 2;
  std::fwrite(stop.data(), 4, n, o);  // rewritten at the end
  int totalSamples = 0;
  for(uint32_t fr = 0; fr < frames; fr++)
  {
    int32_t numSamples;
    if(std::fread(&numSamples, 4, 1, f) != 1 || std::fread(sum.data(), 16, n, f) != n)
      return 2;
    const float total = (float)totalSamples, ns = (float)numSamples, after = (float)(totalSamples + numSamples);
    for(uint32_t i = 0; i < n; i++)
    {
      outM2[i] = outE[i] = NAN;
      if(stop[i])
        continue;
      const float4 c = f4(sum[i].x / ns, sum[i].y / ns, sum[i].z / ns, sum[i].w / ns);
      if(fr == 0)
      {
        img[i] = c;
        m2[i] = 0.0f;
      }
      else
      {
        const float4 old = img[i];
        img[i] = f4((old.x * total + c.x * ns) / after, (old.y * total + c.y * ns) / after, (old.z * total + c.z * ns) / after, (old.w * total + c.w * ns) / after);
        m2[i] = convergeUpdate(m2[i], ns, convergeLum(c), convergeLum(old), convergeLum(img[i]));
      }
      outM2[i] = m2[i];
      outE[i] = convergeRelError(rule, m2[i], fr + 1, after, convergeLum(img[i]));
      if(convergeStops(rule, m2[i], fr + 1, after, convergeLum(img[i])))
        stop[i] = fr + 1;
    }
    totalSamples += numSamples;
    std::fwrite(outM2.data(), 4, n, o);
    std::fwrite(outE.data(), 4, n, o);
  }
  std::fclose(f);
  std::fseek(o, 0, SEEK_SET);
  std::fwrite(stop.data(), 4, n, o);
  std::fclose(o);
  return 0;
}
