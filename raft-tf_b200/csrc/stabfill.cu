// F26: full-frame stabilization -- the flows extended past the frame edge (the residual after each pair's global motion,
// filled by rb_masked_fill) and the warp that fills the borders the corrected camera uncovers from neighbouring frames.
// Every fp32 / fp64 operation is rounded on its own (no FMA contraction), so a numpy restatement reproduces the bits
// (tests/stabfill_oracle.py); no atomics, no allocation.
#include <math.h>

#include "common.cuh"
#include "fb_sample.cuh"

namespace rb {

// The geometry of B flows on the Hn x Wn grid of Hs x Ws frames, extended by my / mx network pixels per side onto the
// Hc x Wc canvas (canvas pixel (i, j) is network position (j - mx, i - my)).
struct ExtGeom {
  double sx, sy, cx, cy, fs;  // Ws / Wn, Hs / Hn, (Ws - 1) / 2, (Hs - 1) / 2, flow_scale
  int Hn, Wn, my, mx, Hc, Wc;
};

// The flow of the similarity m = (a, b, tx, ty) at network position (x, y): the centred frame point p = ((x + 0.5) sx -
// 0.5 - cx, (y + 0.5) sy - 0.5 - cy) moves to M p; (M p - p) in network pixels over flow_scale, in fp64 and rounded once.
__device__ __forceinline__ float2 similarity_flow_at(const double* __restrict__ m, double x, double y, const ExtGeom& g) {
  const double px = __dsub_rn(__dsub_rn(__dmul_rn(__dadd_rn(x, 0.5), g.sx), 0.5), g.cx);
  const double py = __dsub_rn(__dsub_rn(__dmul_rn(__dadd_rn(y, 0.5), g.sy), 0.5), g.cy);
  const double u = __dsub_rn(__dadd_rn(__dsub_rn(__dmul_rn(m[0], px), __dmul_rn(m[1], py)), m[2]), px);
  const double v = __dsub_rn(__dadd_rn(__dadd_rn(__dmul_rn(m[1], px), __dmul_rn(m[0], py)), m[3]), py);
  return make_float2(__double2float_rn(__ddiv_rn(__ddiv_rn(u, g.sx), g.fs)),
                     __double2float_rn(__ddiv_rn(__ddiv_rn(v, g.sy), g.fs)));
}

// finish = 0: the residual r = flow - g inside the grid (hole 0), r = 0 on the band (hole 1).  finish = 1: the extended
// flow, the flow bit for bit inside, r + g on the band (ext may alias resid).  Grid (canvas pixels, B).
__global__ void __launch_bounds__(256) flow_extend_kernel(const float2* __restrict__ flow, const double* __restrict__ motions,
                                                          ExtGeom g, int finish, const float2* resid, float2* out,
                                                          uint8_t* __restrict__ hole) {
  const size_t nc = (size_t)g.Hc * g.Wc;
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nc) return;
  const int b = blockIdx.y;
  const int x = (int)(q % g.Wc) - g.mx, y = (int)(q / g.Wc) - g.my;
  const bool in = x >= 0 && x < g.Wn && y >= 0 && y < g.Hn;
  const size_t o = (size_t)b * nc + q;
  if (in && finish) {
    out[o] = flow[((size_t)b * g.Hn + y) * g.Wn + x];
    return;
  }
  if (!in && !finish) {
    out[o] = make_float2(0.f, 0.f);
    hole[o] = 1;
    return;
  }
  const float2 gf = similarity_flow_at(motions + (size_t)b * 4, (double)x, (double)y, g);
  if (finish) {
    const float2 r = resid[o];
    out[o] = make_float2(__fadd_rn(r.x, gf.x), __fadd_rn(r.y, gf.y));
  } else {
    const float2 f = flow[((size_t)b * g.Hn + y) * g.Wn + x];
    out[o] = make_float2(__fsub_rn(f.x, gf.x), __fsub_rn(f.y, gf.y));
    hole[o] = 0;
  }
}

// The frames' ratios to the network grid, and the Hc x Wc canvas of the extended flows: the grid with my / mx network
// pixels added on each side.
struct FillGeom {
  NetGeom r;
  int Hs, Ws, Hc, Wc, my, mx;
};

// One side of a source outside frame t at canvas position p: up to n chain steps on the extended flows (dir = +1
// forward, -1 backward), stopping when the position leaves the canvas or fails the forward-backward test; found at the
// first frame t + dir n whose own pixels hold the position, unclamped.  Returns the distance (0: not found) and the
// colour.
__device__ __forceinline__ int fill_side(const uint8_t* __restrict__ frames, const float2* __restrict__ fw,
                                         const float2* __restrict__ bw, int t, int dir, int n, float2 p,
                                         const FillGeom& g, float s, float a1, float a2, float* col) {
  const size_t nc = (size_t)g.Hc * g.Wc, ns = (size_t)g.Hs * g.Ws;
  if (!inside_frame(p.x, p.y, g.Hc, g.Wc)) return 0;
  for (int step = 1; step <= n; ++step) {
    const ChainLink l = chain_link(fw, bw, nc, t, dir, step);
    float2 q;
    if (chain_step(l.pull, l.test, g.Hc, g.Wc, s, a1, a2, p, q)) return 0;
    p = q;
    // canvas -> network (exact in fp64) -> frame pixels by the pixel-centre rule, unclamped
    const float ox = __double2float_rn(px_map(__dsub_rn((double)p.x, g.mx), g.r.rxs));
    const float oy = __double2float_rn(px_map(__dsub_rn((double)p.y, g.my), g.r.rys));
    if (!inside_frame(ox, oy, g.Hs, g.Ws)) continue;
    sample_rgb(frames + (size_t)(t + dir * step) * ns * 3, g.Ws, bilerp_at(ox, oy, g.Hs, g.Ws), col);
    return step;
  }
  return 0;
}

// One thread per output pixel, blockIdx.y over the rows (striding); row r = (t, nf, nb) warped by A[r].
__global__ void __launch_bounds__(256) frames_warp_affine_fill_kernel(
    const uint8_t* __restrict__ frames, int F, const float2* __restrict__ fw, const float2* __restrict__ bw, FillGeom g,
    float s, float a1, float a2, const double* __restrict__ A, const int32_t* __restrict__ rows, int n_rows,
    float* __restrict__ colour, uint8_t* __restrict__ status) {
  const int Hs = g.Hs, Ws = g.Ws;
  const size_t ns = (size_t)Hs * Ws;
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= ns) return;
  const double x = (double)(q % (size_t)Ws), y = (double)(q / (size_t)Ws);
  for (int r = blockIdx.y; r < n_rows; r += gridDim.y) {
    const int t = __ldg(rows + 3 * r), nf = __ldg(rows + 3 * r + 1), nb = __ldg(rows + 3 * r + 2);
    float* out = colour + ((size_t)r * ns + q) * 3;
    uint8_t* st = status + (size_t)r * ns + q;
    if (t < 0 || t >= F) {  // an absent row
#pragma unroll
      for (int c = 0; c < 3; ++c) out[c] = 0.f;
      *st = 3;
      continue;
    }
    const double* m = A + (size_t)r * 6;
    const double sx = __dadd_rn(__dadd_rn(__dmul_rn(m[0], x), __dmul_rn(m[1], y)), m[2]);
    const double sy = __dadd_rn(__dadd_rn(__dmul_rn(m[3], x), __dmul_rn(m[4], y)), m[5]);
    const float fx = __double2float_rn(sx), fy = __double2float_rn(sy);
    if (inside_frame(fx, fy, Hs, Ws) || isnan(fx) || isnan(fy)) {  // rb_frames_warp_affine's value before rounding
      const Bilerp bl = bilerp_at(fminf(fmaxf(fx, 0.f), (float)(Ws - 1)), fminf(fmaxf(fy, 0.f), (float)(Hs - 1)), Hs, Ws);
      sample_rgb(frames + (size_t)t * ns * 3, Ws, bl, out);
      *st = 0;
      continue;
    }
    // the source on the canvas: the pixel-centre rule to the network grid (unclamped), shifted by the margin
    const float2 p = make_float2(__double2float_rn(__dadd_rn(px_map(sx, g.r.rxn), (double)g.mx)),
                                 __double2float_rn(__dadd_rn(px_map(sy, g.r.ryn), (double)g.my)));
    float cf[3], cb[3];
    const int df = fill_side(frames, fw, bw, t, 1, min(max(nf, 0), F - 1 - t), p, g, s, a1, a2, cf);
    const int db = fill_side(frames, fw, bw, t, -1, min(max(nb, 0), t), p, g, s, a1, a2, cb);
    blend_sides(df, cf, db, cb, out, st);
  }
}

}  // namespace rb

using namespace rb;

namespace {

int flow_extend(const char* name, const float* flow, const double* motions, int B, int Hn, int Wn, int Hs, int Ws,
                int my, int mx, float flow_scale, int finish, const float* resid, float* out, uint8_t* hole,
                void* stream) {
  RB_REQUIRE(flow && motions && out && (finish ? resid != nullptr : hole != nullptr), RB_ERR_BAD_ARG, "%s: null pointer",
             name);
  RB_REQUIRE(B > 0 && Hn > 0 && Wn > 0 && Hs > 0 && Ws > 0, RB_ERR_BAD_SHAPE,
             "%s: bad shape B=%d Hn=%d Wn=%d Hs=%d Ws=%d", name, B, Hn, Wn, Hs, Ws);
  RB_REQUIRE(my >= 0 && mx >= 0, RB_ERR_BAD_SHAPE, "%s: margins must be >= 0 (got my=%d mx=%d)", name, my, mx);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "%s: flow_scale must be finite and > 0 (got %g)", name, (double)flow_scale);
  const int64_t Hc = (int64_t)Hn + 2 * (int64_t)my, Wc = (int64_t)Wn + 2 * (int64_t)mx;
  RB_REQUIRE(B <= 65535 && Hc < (1 << 24) && Wc < (1 << 24) && Hc * Wc < (int64_t(1) << 31), RB_ERR_BAD_SHAPE,
             "%s: B=%d canvases of %lldx%lld exceed one grid", name, B, (long long)Hc, (long long)Wc);
  RB_REQUIRE((const void*)flow != (const void*)out, RB_ERR_BAD_ARG, "%s: the output must not alias the flow", name);
  ExtGeom g;
  g.sx = (double)Ws / (double)Wn;
  g.sy = (double)Hs / (double)Hn;
  g.cx = 0.5 * (double)(Ws - 1);
  g.cy = 0.5 * (double)(Hs - 1);
  g.fs = (double)flow_scale;
  g.Hn = Hn;
  g.Wn = Wn;
  g.my = my;
  g.mx = mx;
  g.Hc = (int)Hc;
  g.Wc = (int)Wc;
  const size_t nc = (size_t)Hc * Wc;
  flow_extend_kernel<<<dim3((unsigned)((nc + 255) / 256), (unsigned)B), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float2*>(flow), motions, g, finish, reinterpret_cast<const float2*>(resid),
      reinterpret_cast<float2*>(out), hole);
  RB_CHECK_LAUNCH("flow_extend_kernel");
  return RB_OK;
}

}  // namespace

extern "C" int rb_flow_extend_residual(const float* flow, const double* motions, int B, int Hn, int Wn, int Hs, int Ws,
                                       int my, int mx, float flow_scale, float* resid, uint8_t* hole, void* stream) {
  return flow_extend("rb_flow_extend_residual", flow, motions, B, Hn, Wn, Hs, Ws, my, mx, flow_scale, 0, nullptr, resid,
                     hole, stream);
}

extern "C" int rb_flow_extend_finish(const float* flow, const double* motions, int B, int Hn, int Wn, int Hs, int Ws,
                                     int my, int mx, float flow_scale, const float* resid, float* ext, void* stream) {
  return flow_extend("rb_flow_extend_finish", flow, motions, B, Hn, Wn, Hs, Ws, my, mx, flow_scale, 1, resid, ext,
                     nullptr, stream);
}

extern "C" int rb_frames_warp_affine_fill(const uint8_t* frames, int F, int Hs, int Ws, const float* ext_fw,
                                          const float* ext_bw, int Hn, int Wn, int my, int mx, float flow_scale,
                                          float alpha1, float alpha2, const double* A, const int32_t* rows, int n_rows,
                                          float* colour, uint8_t* status, void* stream) {
  const char* fn = "rb_frames_warp_affine_fill";
  if (int rc = check_rows_entry(fn, frames && A && rows && colour && status, ext_fw, ext_bw, F, Hs, Ws, Hn, Wn, n_rows))
    return rc;
  RB_REQUIRE(my >= 0 && mx >= 0, RB_ERR_BAD_SHAPE, "rb_frames_warp_affine_fill: margins must be >= 0 (got my=%d mx=%d)",
             my, mx);
  const int64_t Hc = (int64_t)Hn + 2 * (int64_t)my, Wc = (int64_t)Wn + 2 * (int64_t)mx;
  RB_REQUIRE((size_t)Hs * Ws < (size_t(1) << 31) && Hs < (1 << 24) && Ws < (1 << 24) && Hc < (1 << 24) &&
                 Wc < (1 << 24) && Hc * Wc < (int64_t(1) << 31),
             RB_ERR_BAD_SHAPE, "rb_frames_warp_affine_fill: %dx%d frames or %lldx%lld canvases exceed one grid", Hs, Ws,
             (long long)Hc, (long long)Wc);
  if (int rc = check_rows_step(fn, Hs, Ws, flow_scale, alpha1, alpha2)) return rc;
  const FillGeom g = {net_geom(Hs, Ws, Hn, Wn), Hs, Ws, (int)Hc, (int)Wc, my, mx};
  frames_warp_affine_fill_kernel<<<rows_grid(Hs, Ws, 256, n_rows), 256, 0, (cudaStream_t)stream>>>(
      frames, F, reinterpret_cast<const float2*>(ext_fw), reinterpret_cast<const float2*>(ext_bw), g, flow_scale, alpha1,
      alpha2, A, rows, n_rows, colour, status);
  RB_CHECK_LAUNCH("frames_warp_affine_fill_kernel");
  return RB_OK;
}
