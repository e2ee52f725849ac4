// host_caps_check.cpp — the alpha-cap bake (../alpha_caps.cuh: capBakeCell, the code k_cap_bake runs per cell) compiled for the host
// through host_shim.h, on records written by tests/test_alpha_caps.py.
//   host_caps_check in.bin out.bin [holes]
//   in:  u32 n, then n records: f32 uv[6], i32 w, h, wrapS, wrapT, f32 factor, cutoff, u32 modeFlags, colA, hasTexture,
//        then (hasTexture) w * h alpha bytes, row-major
//   out: n x kCapWords u32, the cap bits of every record (bit i = micro-triangle i in ommBary2Index order); with `holes` its hole bits
#include "host_shim.h"

#include <cstdio>
#include <cstring>
#include <vector>

#include "../alpha_caps.cuh"

using namespace pt;

// the sampler's wrap of an integer texel coordinate (glTF REPEAT / CLAMP_TO_EDGE / MIRRORED_REPEAT, as shade.cuh's wrapCoord)
static int wrapHost(int i, int n, int mode)
{
  if(mode == 33071)
    return i < 0 ? 0 : (i > n - 1 ? n - 1 : i);
  if(mode == 33648)
  {
    const int p = 2 * n, m = ((i % p) + p) % p;
    return m < n ? m : p - 1 - m;
  }
  return ((i % n) + n) % n;
}

int main(int argc, char** argv)
{
  if(argc < 3)
    return 2;
  const bool holes = argc > 3 && std::strcmp(argv[3], "holes") == 0;
  FILE* f = std::fopen(argv[1], "rb");
  FILE* o = std::fopen(argv[2], "wb");
  if(!f || !o)
    return 2;
  uint32_t n = 0;
  if(std::fread(&n, 4, 1, f) != 1)
    return 2;
  for(uint32_t r = 0; r < n; r++)
  {
    float    uv[6], fc[2];
    int32_t  dims[4];
    uint32_t flags[3];
    if(std::fread(uv, 4, 6, f) != 6 || std::fread(dims, 4, 4, f) != 4 || std::fread(fc, 4, 2, f) != 2 || std::fread(flags, 4, 3, f) != 3)
      return 2;
    const int            w = dims[0], h = dims[1];
    std::vector<uint8_t> alpha(flags[2] ? (size_t)w * h : 0);
    if(!alpha.empty() && std::fread(alpha.data(), 1, alpha.size(), f) != alpha.size())
      return 2;
    auto                  alpha8 = [&](int x, int y) { return (int)alpha[(size_t)y * w + x]; };
    const uint32_t        wrapBits = ((uint32_t)dims[2] & 0xffffu) | ((uint32_t)dims[3] << 16);
    std::vector<uint32_t> bits(kCapWords, 0u);
    for(uint32_t k = 0; k < 2 * kCapMicro; k++)
    {
      uint32_t idx;
      bool     cap, hole;
      if(capBakeCell(k, uv, w, h, wrapBits, fc[0], fc[1], flags[0], flags[1], flags[2] != 0, alpha8, wrapHost, idx, cap, hole) && (holes ? hole : cap))
        bits[idx >> 5] |= 1u << (idx & 31u);
    }
    std::fwrite(bits.data(), 4, bits.size(), o);
  }
  std::fclose(f);
  std::fclose(o);
  return 0;
}
