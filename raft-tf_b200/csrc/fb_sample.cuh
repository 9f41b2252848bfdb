// The bilinear flow sample and the forward-backward test of F5 (csrc/consistency.cu), shared by every kernel that must
// reproduce rb_flow_fb_check's bits: the per-pixel check and the point tracker (csrc/track.cu).  Every operation is rounded
// on its own, left to right (__fmul_rn / __fadd_rn / __fsub_rn: no FMA contraction), so an fp32 restatement in numpy
// reproduces them exactly (tests/fb_oracle.py, tests/track_oracle.py).
#pragma once

#include <math.h>

#include "common.cuh"

namespace rb {

// Bilinear weights of a point q inside [0, W-1] x [0, H-1] (the caller checks that): the four taps and their weights.
struct Bilerp {
  int x0, x1, y0, y1;
  float ax, ay, cx, cy;
};

__device__ __forceinline__ Bilerp bilerp_at(float qx, float qy, int H, int W) {
  Bilerp b;
  b.x0 = (int)floorf(qx);
  b.y0 = (int)floorf(qy);
  b.x1 = min(b.x0 + 1, W - 1);
  b.y1 = min(b.y0 + 1, H - 1);
  b.ax = __fsub_rn(qx, (float)b.x0);
  b.ay = __fsub_rn(qy, (float)b.y0);
  b.cx = __fsub_rn(1.f, b.ax);
  b.cy = __fsub_rn(1.f, b.ay);
  return b;
}

// ((1-ax) v00 + ax v01)(1-ay) + ((1-ax) v10 + ax v11) ay of one channel
__device__ __forceinline__ float bilerp1(const Bilerp& b, float v00, float v01, float v10, float v11) {
  const float t0 = __fadd_rn(__fmul_rn(b.cx, v00), __fmul_rn(b.ax, v01));
  const float t1 = __fadd_rn(__fmul_rn(b.cx, v10), __fmul_rn(b.ax, v11));
  return __fadd_rn(__fmul_rn(t0, b.cy), __fmul_rn(t1, b.ay));
}

// s times the bilinear sample of the [H,W] float2 field img at the taps of b
__device__ __forceinline__ float2 sample_flow(const float2* __restrict__ img, int W, const Bilerp& b, float s) {
  const float2 v00 = img[(size_t)b.y0 * W + b.x0], v01 = img[(size_t)b.y0 * W + b.x1];
  const float2 v10 = img[(size_t)b.y1 * W + b.x0], v11 = img[(size_t)b.y1 * W + b.x1];
  return make_float2(__fmul_rn(s, bilerp1(b, v00.x, v01.x, v10.x, v11.x)),
                     __fmul_rn(s, bilerp1(b, v00.y, v01.y, v10.y, v11.y)));
}

// x' = fl32((x + 0.5) r - 0.5) in fp64, each operation rounded on its own, clamped into [0, n - 1]: the pixel-centre map
// between the network grid and a frame's own pixels (r = n_to / n_from)
__device__ __forceinline__ float px_remap(double x, double r, int n) {
  const float v = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn(x, 0.5), r), 0.5));
  return fminf(fmaxf(v, 0.f), (float)(n - 1));
}

// Whether q = p + f lies inside [0, W-1] x [0, H-1]; written so that a NaN coordinate counts as outside.
__device__ __forceinline__ bool inside_frame(float qx, float qy, int H, int W) {
  return qx >= 0.f && qx <= (float)(W - 1) && qy >= 0.f && qy <= (float)(H - 1);
}

// The test of a forward step f and the backward flow b sampled at its target: 1 if |f+b|^2 > a1 (|f|^2 + |b|^2) + a2
// (inconsistent, occluded), else 0.
__device__ __forceinline__ uint8_t fb_inconsistent(float2 f, float2 b, float a1, float a2) {
  const float ex = __fadd_rn(f.x, b.x), ey = __fadd_rn(f.y, b.y);
  const float d = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey));
  const float mag =
      __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(f.x, f.x), __fmul_rn(f.y, f.y)), __fmul_rn(b.x, b.x)), __fmul_rn(b.y, b.y));
  const float m = __fadd_rn(__fmul_rn(a1, mag), a2);
  return d > m ? 1 : 0;
}

}  // namespace rb
