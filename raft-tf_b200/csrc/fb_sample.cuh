// The bilinear flow sample and the forward-backward test of F5 (csrc/consistency.cu), and the chain step built on them:
// one link of a pixel followed through consecutive flows.  Every kernel that must reproduce rb_flow_fb_check's bits
// uses them: the per-pixel check, the flow accumulation (csrc/propagate.cu), the point trackers (csrc/track.cu), object
// removal (csrc/inpaint.cu), full-frame stabilization (csrc/stabfill.cu), denoising (csrc/denoise.cu), temporal
// consistency and the warping error (csrc/temporal.cu) and motion segmentation (csrc/motionseg.cu).  Every operation is
// rounded on its own, left to right (__fmul_rn / __fadd_rn / __fsub_rn: no FMA contraction), so an fp32 restatement in
// numpy reproduces them exactly (tests/fb_oracle.py, tests/track_oracle.py and the oracles of those kernels).
#pragma once

#include <math.h>

#include <algorithm>

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

// Channel c of the bilinear sample of the [.,W,3] uint8 image img at the taps of b
__device__ __forceinline__ float sample_rgb1(const uint8_t* __restrict__ img, int W, const Bilerp& b, int c) {
  const size_t r0 = (size_t)b.y0 * W, r1 = (size_t)b.y1 * W;
  return bilerp1(b, (float)img[(r0 + b.x0) * 3 + c], (float)img[(r0 + b.x1) * 3 + c], (float)img[(r1 + b.x0) * 3 + c],
                 (float)img[(r1 + b.x1) * 3 + c]);
}

// All three channels of that sample
__device__ __forceinline__ void sample_rgb(const uint8_t* __restrict__ img, int W, const Bilerp& b, float* col) {
#pragma unroll
  for (int c = 0; c < 3; ++c) col[c] = sample_rgb1(img, W, b, c);
}

// The ratios between a frame's own Hs x Ws pixels and the Hn x Wn network grid of its flows.
struct NetGeom {
  double rxn, ryn, rxs, rys;  // Wn / Ws, Hn / Hs, Ws / Wn, Hs / Hn
};

inline NetGeom net_geom(int Hs, int Ws, int Hn, int Wn) {
  NetGeom g;
  g.rxn = (double)Wn / (double)Ws;
  g.ryn = (double)Hn / (double)Hs;
  g.rxs = (double)Ws / (double)Wn;
  g.rys = (double)Hs / (double)Hn;
  return g;
}

// (x + 0.5) r - 0.5 in fp64, each operation rounded on its own: the pixel-centre map between the network grid and a
// frame's own pixels (r = n_to / n_from, a ratio of NetGeom)
__device__ __forceinline__ double px_map(double x, double r) { return __dsub_rn(__dmul_rn(__dadd_rn(x, 0.5), r), 0.5); }

// px_map rounded to fp32 and clamped into [0, n - 1] (track_queries / tracks_to_frames)
__device__ __forceinline__ float px_remap(double x, double r, int n) {
  const float v = __double2float_rn(px_map(x, r));
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

// One link of a chain on the H x W grid from p inside it: f = s pull(p), q = p + f.  Returns 2 when q leaves the grid
// (or is NaN), else F5's test of f against s test(q): 0 consistent, 1 not.
__device__ __forceinline__ uint8_t chain_step(const float2* __restrict__ pull, const float2* __restrict__ test, int H,
                                              int W, float s, float a1, float a2, float2 p, float2& q) {
  const float2 f = sample_flow(pull, W, bilerp_at(p.x, p.y, H, W), s);
  q = make_float2(__fadd_rn(p.x, f.x), __fadd_rn(p.y, f.y));
  if (!inside_frame(q.x, q.y, H, W)) return 2;
  return fb_inconsistent(f, sample_flow(test, W, bilerp_at(q.x, q.y, H, W), s), a1, a2);
}

// The flows of link `step` of a chain from frame t through consecutive [npix] fields: dir = +1 pulls with fw[t+step-1]
// and tests against bw; dir = -1 is the mirror, pulling with bw[t-step] and testing against fw.
struct ChainLink {
  const float2* pull;
  const float2* test;
};

__device__ __forceinline__ ChainLink chain_link(const float2* fw, const float2* bw, size_t npix, int t, int dir,
                                                int step) {
  const size_t k = (size_t)(dir > 0 ? t + step - 1 : t - step) * npix;
  return dir > 0 ? ChainLink{fw + k, bw + k} : ChainLink{bw + k, fw + k};
}

// The two sides of a pixel, found df and db frames away (0: not found) with colours cf and cb, blended toward the nearer
// frame: (db cf + df cb) / (df + db) and status 1 with both, the side found and status 2 with one, 0 and status 3 with none.
__device__ __forceinline__ void blend_sides(int df, const float* cf, int db, const float* cb, float* out,
                                            uint8_t* status) {
  if (df && db) {
    const float wf = (float)db, wb = (float)df, den = (float)(df + db);
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = __fdiv_rn(__fadd_rn(__fmul_rn(wf, cf[c]), __fmul_rn(wb, cb[c])), den);
    *status = 1;
  } else if (df || db) {
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = df ? cf[c] : cb[c];
    *status = 2;
  } else {
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c] = 0.f;
    *status = 3;
  }
}

// ---- host side of the row-table entries (rb_inpaint_propagate, rb_denoise_merge, rb_frames_warp_affine_fill,
// rb_motion_segment): F frames, Hn x Wn flows, one output row per (t, nf, nb) ----

// Their first checks, each message prefixed by fn: the entry's own pointers (ptrs), the flows (null only when F < 2),
// the shapes.
inline int check_rows_entry(const char* fn, bool ptrs, const void* flow_fw, const void* flow_bw, int F, int Hs, int Ws,
                            int Hn, int Wn, int n_rows) {
  RB_REQUIRE(ptrs && (F < 2 || (flow_fw && flow_bw)), RB_ERR_BAD_ARG, "%s: null pointer", fn);
  RB_REQUIRE(F > 0 && Hs > 0 && Ws > 0 && Hn > 0 && Wn > 0 && n_rows > 0, RB_ERR_BAD_SHAPE,
             "%s: bad shape F=%d Hs=%d Ws=%d Hn=%d Wn=%d n_rows=%d", fn, F, Hs, Ws, Hn, Wn, n_rows);
  return RB_OK;
}

// Their last checks: Hs x Ws pixels per frame inside one grid, and the flow scale and F5's alphas.  An entry checks its
// own shape arguments between the two (rb_frames_warp_affine_fill: the margins and the canvas).
inline int check_rows_step(const char* fn, int Hs, int Ws, float flow_scale, float alpha1, float alpha2) {
  RB_REQUIRE((size_t)Hs * Ws < (size_t(1) << 31), RB_ERR_BAD_SHAPE, "%s: %dx%d pixels per frame exceed one grid", fn, Hs,
             Ws);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "%s: flow_scale must be finite and > 0 (got %g)", fn, (double)flow_scale);
  RB_REQUIRE(alpha1 >= 0.f && isfinite(alpha1) && alpha2 >= 0.f && isfinite(alpha2), RB_ERR_BAD_ARG,
             "%s: alpha1, alpha2 must be finite and >= 0 (got %g, %g)", fn, (double)alpha1, (double)alpha2);
  return RB_OK;
}

// Their grid: blocks of `threads` frame pixels x up to 65535 rows (the kernels stride blockIdx.y over the rest).
inline dim3 rows_grid(int Hs, int Ws, int threads, int n_rows) {
  const size_t ns = (size_t)Hs * Ws;
  return dim3((unsigned)((ns + threads - 1) / threads), (unsigned)std::min(n_rows, 65535));
}

}  // namespace rb
