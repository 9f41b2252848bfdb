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

struct FillGeom {
  double rxn, ryn, rxs, rys;  // Wn / Ws, Hn / Hs, Ws / Wn, Hs / Hn
  int Hs, Ws, Hc, Wc, my, mx;
};

// One side of a source outside frame t at canvas position p: up to n steps of rb_track_points' step on the extended
// flows (dir = +1: pull with fw, test against bw; -1: the mirror), stopping when the position leaves the canvas or fails
// the forward-backward test; found at the first frame t + dir n whose own pixels hold the position, unclamped.  Returns
// the distance (0: not found) and the colour.
__device__ __forceinline__ int fill_side(const uint8_t* __restrict__ frames, const float2* __restrict__ fw,
                                         const float2* __restrict__ bw, int t, int dir, int n, float2 p,
                                         const FillGeom& g, float s, float a1, float a2, float* col) {
  const size_t nc = (size_t)g.Hc * g.Wc, ns = (size_t)g.Hs * g.Ws;
  if (!inside_frame(p.x, p.y, g.Hc, g.Wc)) return 0;
  for (int step = 1; step <= n; ++step) {
    const size_t k = (size_t)(dir > 0 ? t + step - 1 : t - step) * nc;
    const float2* pull = (dir > 0 ? fw : bw) + k;
    const float2* test = (dir > 0 ? bw : fw) + k;
    const float2 f = sample_flow(pull, g.Wc, bilerp_at(p.x, p.y, g.Hc, g.Wc), s);
    const float2 q = make_float2(__fadd_rn(p.x, f.x), __fadd_rn(p.y, f.y));
    if (!inside_frame(q.x, q.y, g.Hc, g.Wc)) return 0;
    if (fb_inconsistent(f, sample_flow(test, g.Wc, bilerp_at(q.x, q.y, g.Hc, g.Wc), s), a1, a2)) return 0;
    p = q;
    // canvas -> network (exact in fp64) -> frame pixels by the pixel-centre rule, unclamped
    const float ox = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dsub_rn((double)p.x, g.mx), 0.5), g.rxs), 0.5));
    const float oy = __double2float_rn(__dsub_rn(__dmul_rn(__dadd_rn(__dsub_rn((double)p.y, g.my), 0.5), g.rys), 0.5));
    if (!inside_frame(ox, oy, g.Hs, g.Ws)) continue;
    const Bilerp b = bilerp_at(ox, oy, g.Hs, g.Ws);
    const uint8_t* img = frames + (size_t)(t + dir * step) * ns * 3;
    const size_t i00 = ((size_t)b.y0 * g.Ws + b.x0) * 3, i01 = ((size_t)b.y0 * g.Ws + b.x1) * 3;
    const size_t i10 = ((size_t)b.y1 * g.Ws + b.x0) * 3, i11 = ((size_t)b.y1 * g.Ws + b.x1) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c)
      col[c] = bilerp1(b, (float)img[i00 + c], (float)img[i01 + c], (float)img[i10 + c], (float)img[i11 + c]);
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
      const uint8_t* img = frames + (size_t)t * ns * 3;
      const size_t i00 = ((size_t)bl.y0 * Ws + bl.x0) * 3, i01 = ((size_t)bl.y0 * Ws + bl.x1) * 3;
      const size_t i10 = ((size_t)bl.y1 * Ws + bl.x0) * 3, i11 = ((size_t)bl.y1 * Ws + bl.x1) * 3;
#pragma unroll
      for (int c = 0; c < 3; ++c)
        out[c] = bilerp1(bl, (float)img[i00 + c], (float)img[i01 + c], (float)img[i10 + c], (float)img[i11 + c]);
      *st = 0;
      continue;
    }
    // the source on the canvas: the pixel-centre rule to the network grid (unclamped), shifted by the margin
    const float2 p = make_float2(
        __double2float_rn(__dadd_rn(__dsub_rn(__dmul_rn(__dadd_rn(sx, 0.5), g.rxn), 0.5), (double)g.mx)),
        __double2float_rn(__dadd_rn(__dsub_rn(__dmul_rn(__dadd_rn(sy, 0.5), g.ryn), 0.5), (double)g.my)));
    float cf[3], cb[3];
    const int df = fill_side(frames, fw, bw, t, 1, min(max(nf, 0), F - 1 - t), p, g, s, a1, a2, cf);
    const int db = fill_side(frames, fw, bw, t, -1, min(max(nb, 0), t), p, g, s, a1, a2, cb);
    if (df && db) {
      const float wf = (float)db, wb = (float)df, den = (float)(df + db);
#pragma unroll
      for (int c = 0; c < 3; ++c) out[c] = __fdiv_rn(__fadd_rn(__fmul_rn(wf, cf[c]), __fmul_rn(wb, cb[c])), den);
      *st = 1;
    } else if (df || db) {
#pragma unroll
      for (int c = 0; c < 3; ++c) out[c] = df ? cf[c] : cb[c];
      *st = 2;
    } else {
#pragma unroll
      for (int c = 0; c < 3; ++c) out[c] = 0.f;
      *st = 3;
    }
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
  RB_REQUIRE(frames && A && rows && colour && status && (F < 2 || (ext_fw && ext_bw)), RB_ERR_BAD_ARG,
             "rb_frames_warp_affine_fill: null pointer");
  RB_REQUIRE(F > 0 && Hs > 0 && Ws > 0 && Hn > 0 && Wn > 0 && n_rows > 0, RB_ERR_BAD_SHAPE,
             "rb_frames_warp_affine_fill: bad shape F=%d Hs=%d Ws=%d Hn=%d Wn=%d n_rows=%d", F, Hs, Ws, Hn, Wn, n_rows);
  RB_REQUIRE(my >= 0 && mx >= 0, RB_ERR_BAD_SHAPE, "rb_frames_warp_affine_fill: margins must be >= 0 (got my=%d mx=%d)",
             my, mx);
  const int64_t Hc = (int64_t)Hn + 2 * (int64_t)my, Wc = (int64_t)Wn + 2 * (int64_t)mx;
  RB_REQUIRE((size_t)Hs * Ws < (size_t(1) << 31) && Hs < (1 << 24) && Ws < (1 << 24) && Hc < (1 << 24) &&
                 Wc < (1 << 24) && Hc * Wc < (int64_t(1) << 31),
             RB_ERR_BAD_SHAPE, "rb_frames_warp_affine_fill: %dx%d frames or %lldx%lld canvases exceed one grid", Hs, Ws,
             (long long)Hc, (long long)Wc);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "rb_frames_warp_affine_fill: flow_scale must be finite and > 0 (got %g)", (double)flow_scale);
  RB_REQUIRE(alpha1 >= 0.f && isfinite(alpha1) && alpha2 >= 0.f && isfinite(alpha2), RB_ERR_BAD_ARG,
             "rb_frames_warp_affine_fill: alpha1, alpha2 must be finite and >= 0 (got %g, %g)", (double)alpha1,
             (double)alpha2);
  FillGeom g;
  g.rxn = (double)Wn / (double)Ws;
  g.ryn = (double)Hn / (double)Hs;
  g.rxs = (double)Ws / (double)Wn;
  g.rys = (double)Hs / (double)Hn;
  g.Hs = Hs;
  g.Ws = Ws;
  g.Hc = (int)Hc;
  g.Wc = (int)Wc;
  g.my = my;
  g.mx = mx;
  const size_t ns = (size_t)Hs * Ws;
  const dim3 grid((unsigned)((ns + 255) / 256), (unsigned)std::min(n_rows, 65535));
  frames_warp_affine_fill_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(
      frames, F, reinterpret_cast<const float2*>(ext_fw), reinterpret_cast<const float2*>(ext_bw), g, flow_scale, alpha1,
      alpha2, A, rows, n_rows, colour, status);
  RB_CHECK_LAUNCH("frames_warp_affine_fill_kernel");
  return RB_OK;
}
