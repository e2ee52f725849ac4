// host_shim.h — lets g++ compile the DEVICE traversal code (../traverse.cuh, ../vec.cuh) for the host, one "lane" at a
// time, so that the exact source the sm_90a kernels run can be checked against brute force without a GPU
// (tools/host_traverse_check.cpp, tests/test_device_source_on_host.py).  Only what traverse.cuh uses is provided.
#pragma once
#include <cuda_runtime.h>  // vector types; __host__ / __device__ expand to nothing outside nvcc

#include <cmath>
#include <cstdint>
#include <cstring>

#ifndef __CUDACC__
#ifndef __forceinline__
#define __forceinline__ inline
#endif
#ifndef __noinline__
#define __noinline__ __attribute__((noinline))
#endif
static inline uint32_t __float_as_uint(float f) { uint32_t u; std::memcpy(&u, &f, 4); return u; }
static inline float    __uint_as_float(uint32_t u) { float f; std::memcpy(&f, &u, 4); return f; }
static inline int      __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline float    __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
static inline int      __clz(uint32_t x) { return x ? __builtin_clz(x) : 32; }
static inline int      __popc(uint32_t x) { return __builtin_popcount(x); }
template <typename T>
static inline T __ldg(const T* p) { return *p; }
using std::isnan;
using std::isinf;
// sequential stand-ins for the atomics of the build kernels (the host harness runs the "threads" one after another)
template <typename T>
static inline T atomicAdd(T* p, T v) { const T o = *p; *p = o + v; return o; }
static inline int atomicMin(int* p, int v) { const int o = *p; if(v < o) *p = v; return o; }
static inline int atomicMax(int* p, int v) { const int o = *p; if(v > o) *p = v; return o; }
// one lane per "warp"
static inline unsigned __activemask() { return 1u; }
static inline unsigned __ballot_sync(unsigned, int pred) { return pred ? 1u : 0u; }
#endif
