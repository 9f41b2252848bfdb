// The per-pixel arithmetic of cv2's float32 bilinear resize, shared by rb_frames_resize / rb_flow_resize (resize.cu) and
// the resized frame synthesis (interp.cu), so that a flow resized inside the blend has the bits of rb_flow_resize.
// tests/resize_oracle.py restates it.
#pragma once
#include "common.cuh"

namespace rb {

enum { RS_COPY = 0, RS_OPENCV = 1, RS_IPP = 2 };

// OpenCV's per-axis coordinate (resize.cpp, resizeGeneric): f = fl32((d + 0.5) * scale - 0.5), scale = 1 / (dst / src)
__device__ __forceinline__ void cv_coord(int d, double scale, int& s, float& f) {
  const float c = __double2float_rn(__dadd_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), -0.5));
  const float fl = floorf(c);
  s = (int)fl;
  f = __fsub_rn(c, fl);
}

// IPP's per-axis coordinate: c = (d + 0.5) * (src / dst) - 0.5 in float64, weight fl32(c - floor(c))
__device__ __forceinline__ void ipp_coord(int d, double scale, int src, int& i0, int& i1, float& w) {
  const double c = __dadd_rn(__dmul_rn(__dadd_rn((double)d, 0.5), scale), -0.5);
  const double fl = floor(c);
  w = __double2float_rn(__dsub_rn(c, fl));
  const int s = (int)fl;
  i0 = min(max(s, 0), src - 1);
  i1 = min(max(s + 1, 0), src - 1);
}

__device__ __forceinline__ float lerp_fma(float p0, float p1, float w) { return __fmaf_rn(w, __fsub_rn(p1, p0), p0); }

// float32 resize of pixel (y, x) of one channel-interleaved [H,W,C] plane, as cv2 computes it (mode RS_*)
template <int C>
__device__ __forceinline__ void resize_f32_px(const float* __restrict__ p, int H, int W, int Ho, int Wo, int y, int x,
                                              int mode, float out[C]) {
  if (mode == RS_COPY) {
#pragma unroll
    for (int c = 0; c < C; ++c) out[c] = p[((size_t)y * W + x) * C + c];
    return;
  }
  if (mode == RS_IPP) {
    int x0, x1, y0, y1;
    float wx, wy;
    ipp_coord(x, (double)W / Wo, W, x0, x1, wx);
    ipp_coord(y, (double)H / Ho, H, y0, y1, wy);
    // IPP's border strips: a column whose taps clamping merged copies its pixel (rows likewise), but the corners run
    // the general formula -- only visible with inf / NaN inputs, where inf - inf gives NaN
    const bool cx = x0 == x1, cy = y0 == y1;
    const float *r0 = p + (size_t)y0 * W * C, *r1 = p + (size_t)y1 * W * C;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      float h0, h1;
      if (cx && !cy) {
        h0 = r0[x0 * C + c];
        h1 = r1[x0 * C + c];
      } else {
        h0 = lerp_fma(r0[x0 * C + c], r0[x1 * C + c], wx);
        h1 = lerp_fma(r1[x0 * C + c], r1[x1 * C + c], wx);
      }
      out[c] = (cy && !cx) ? h0 : lerp_fma(h0, h1, wy);
    }
    return;
  }
  // RS_OPENCV: OpenCV's own float code (single-row or single-column sources)
  int sx, sy;
  float fx, fy;
  cv_coord(x, 1.0 / ((double)Wo / W), sx, fx);
  cv_coord(y, 1.0 / ((double)Ho / H), sy, fy);
  if (sx < 0) { sx = 0; fx = 0.f; }
  if (sx >= W - 1) { sx = W - 1; fx = 0.f; }
  const bool one_tap = sx >= W - 1;  // OpenCV's xmax: from there on S[sx] alone
  const int x0 = sx, x1 = min(sx + 1, W - 1);
  const int y0 = min(max(sy, 0), H - 1), y1 = min(max(sy + 1, 0), H - 1);
  const float a0 = __fsub_rn(1.f, fx), b0 = __fsub_rn(1.f, fy);
  const float *r0 = p + (size_t)y0 * W * C, *r1 = p + (size_t)y1 * W * C;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const float h0 = one_tap ? r0[x0 * C + c] : __fadd_rn(__fmul_rn(r0[x0 * C + c], a0), __fmul_rn(r0[x1 * C + c], fx));
    const float h1 = one_tap ? r1[x0 * C + c] : __fadd_rn(__fmul_rn(r1[x0 * C + c], a0), __fmul_rn(r1[x1 * C + c], fx));
    out[c] = __fadd_rn(__fmul_rn(h0, b0), __fmul_rn(h1, fy));
  }
}

__host__ __device__ inline int float_mode(int H, int W, int Ho, int Wo) {
  return (H == Ho && W == Wo) ? RS_COPY : (H == 1 || W == 1) ? RS_OPENCV : RS_IPP;
}

// The H x W network pixel whose area holds the centre of Hs x Ws output pixel (x, y): (((2x+1) W) div (2 Ws),
// ((2y+1) H) div (2 Hs)), as a raster index
__device__ __forceinline__ size_t near_px(int x, int y, int H, int W, int Hs, int Ws) {
  return (size_t)(((2 * (uint64_t)y + 1) * (uint64_t)H) / (2 * (uint64_t)Hs)) * W +
         (size_t)(((2 * (uint64_t)x + 1) * (uint64_t)W) / (2 * (uint64_t)Ws));
}

// resize_flow's factors u *= dW / float(W_), v *= dH / float(H_): the float64 quotient rounded to fp32 (numpy >= 2,
// float32 array)
inline float flow_scale_u(int W, int Wo) { return (float)((double)Wo / (double)W); }
inline float flow_scale_v(int H, int Ho) { return (float)((double)Ho / (double)H); }

}  // namespace rb
