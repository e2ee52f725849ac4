// converge.cuh — the per-pixel stopping rule of b200pt_set_convergence (DESIGN.md §2 "Convergence"), one source for the
// device (k_accumulate<true>), the library's host read-back (b200pt_read_convergence) and the host check
// (tools/host_converge_check.cpp).
//
// An accumulation starts at a frame carrying B200PT_PT_FIRST_FRAME.  For an active pixel, every frame f folds the luminance
// c_f of its clamped sample mean into the running mean m with weight n_f = numSamples, and West's weighted Welford update
//   M2 += n_f (c_f - m_prev)(c_f - m)
// keeps the weighted sum of squares; E[M2] = (F - 1) sigma^2 for F frames of i.i.d. samples, whatever the n_f.  The relative
// standard error of the pixel's mean after N = sum n_f samples is then
//   e = sqrt(M2 / ((F - 1) N)) / max(m, floor)      (+inf while F < 2).
// At a checkpoint (F a multiple of `interval`) an active pixel with F >= minFrames and e <= threshold stops for the rest of the
// accumulation.  Every active pixel has the same F and N, so the state per pixel is M2 and the frame count at which it stopped.
#pragma once
#include "vec.cuh"

namespace pt {

struct ConvergeRule
{
  float    threshold;  // > 0
  float    floor;      // >= 0: the luminance below which the error is taken relative to `floor`
  uint32_t minFrames;  // >= 2
  uint32_t interval;   // >= 1
};

PT_HD float convergeLum(float4 c) { return (c.x + c.y + c.z) * (1.0f / 3.0f); }

// one frame of an active pixel: c its frame's luminance, weight n, mPrev / m the running mean's luminance before / after the frame
PT_HD float convergeUpdate(float m2, float n, float c, float mPrev, float m) { return m2 + n * (c - mPrev) * (c - m); }

// e after `frames` frames and `samples` samples.  M2 is clamped at 0: each term (c - m_prev)(c - m) is >= 0 in exact arithmetic, but
// with c close to m_prev the rounded mean can land on the far side of c and a flat pixel's M2 can go slightly negative.  With
// floor 0, a pixel whose mean luminance is 0 has e = 0 / 0 = NaN and never stops (include/b200pt.h).
PT_HD float convergeRelError(const ConvergeRule& r, float m2, uint32_t frames, float samples, float m)
{
  if(frames < 2u)
    return INFINITY;
  return sqrtf(fmaxf(m2, 0.0f) / ((float)(frames - 1u) * samples)) / fmaxf(m, r.floor);
}

// the decision after frame `frames` of an active pixel: it stops only at a checkpoint past minFrames
PT_HD bool convergeStops(const ConvergeRule& r, float m2, uint32_t frames, float samples, float m)
{
  return frames % r.interval == 0u && frames >= r.minFrames && convergeRelError(r, m2, frames, samples, m) <= r.threshold;
}

}  // namespace pt
