// F22 / F23: video stabilization -- a robust similarity fit of each frame pair's camera motion to its flow, and the warp
// of every frame by its correction at the frame's own size.
#include <math.h>

#include "common.cuh"
#include "fb_sample.cuh"

namespace rb {

constexpr int kGmThreads = 256;
constexpr int kGmPerThread = 16;
constexpr int kGmChunk = kGmThreads * kGmPerThread;  // pixels per block
constexpr int kGmSums = RB_MOTION_SUMS;
// a system is singular when the weighted spread of the points is below this fraction of their weighted mean |p|^2
constexpr double kGmSingular = 1e-9;

// The frames' geometry, shared by every pixel: network pixel (i, j) sits at ((j + 0.5) sx - 0.5 - cx, (i + 0.5) sy -
// 0.5 - cy) in centred frame pixels, and a flow (u, v) moves it by fs (u sx, v sy).
struct GmGeom {
  double sx, sy, cx, cy, isx, isy, fs, inv_c2;
};

// Fixed-shape tree over the block for all the sums at once: s[k][t] += s[k][t + h] for h = 128, 64, ..., 1.
__device__ __forceinline__ void gm_block_sum(double (*s)[kGmThreads]) {
  const int t = threadIdx.x;
  __syncthreads();
#pragma unroll
  for (int h = kGmThreads / 2; h > 0; h >>= 1) {
    if (t < h) {
#pragma unroll
      for (int k = 0; k < kGmSums; ++k) s[k][t] += s[k][t + h];
    }
    __syncthreads();
  }
}

// 1 / d for a finite d >= 1 to within an ulp: the hardware's approximate fp64 reciprocal refined by two Newton steps
// (the correctly rounded division calls a slow path that makes ptxas spill in the pixel loop).
__device__ __forceinline__ double recip_ge1(double d) {
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
  y = fma(y, fma(-d, y, 1.0), y);
  return fma(y, fma(-d, y, 1.0), y);
}

// grid (chunks per pair, B); thread t takes pixels chunk_start + k * 256 + t, k = 0..15 in order (coalesced).  Round 0
// (params NULL) weighs every pixel with occ == 0 and a finite flow by 1; a later round by 1 / (1 + (r / c)^2), r the
// residual of the previous round's similarity in network pixels.
__global__ void __launch_bounds__(kGmThreads) global_motion_chunk_kernel(const float2* __restrict__ flow,
                                                                         const uint8_t* __restrict__ occ, int Wn,
                                                                         size_t npix, GmGeom g,
                                                                         const double* __restrict__ params,
                                                                         double* __restrict__ partials) {
  __shared__ double red[kGmSums][kGmThreads];
  const int b = blockIdx.y;
  const size_t base = (size_t)b * npix;
  const size_t c0 = (size_t)blockIdx.x * kGmChunk;
  double m0 = 1.0, m1 = 0.0, m2 = 0.0, m3 = 0.0;
  if (params) {
    m0 = params[(size_t)b * 4 + 0];
    m1 = params[(size_t)b * 4 + 1];
    m2 = params[(size_t)b * 4 + 2];
    m3 = params[(size_t)b * 4 + 3];
  }
  double v[kGmSums];
#pragma unroll
  for (int k = 0; k < kGmSums; ++k) v[k] = 0.0;
  for (int k = 0; k < kGmPerThread; ++k) {
    const size_t q = c0 + (size_t)k * kGmThreads + threadIdx.x;
    if (q >= npix) break;
    const size_t p = base + q;
    const float2 f = flow[p];
    if (occ[p] != 0 || !isfinite(f.x) || !isfinite(f.y)) continue;
    const int i = (int)q / Wn, j = (int)q % Wn;  // npix < 2^31
    const double px = ((double)j + 0.5) * g.sx - 0.5 - g.cx, py = ((double)i + 0.5) * g.sy - 0.5 - g.cy;
    const double qx = px + g.fs * ((double)f.x * g.sx), qy = py + g.fs * ((double)f.y * g.sy);
    double w = 1.0;
    if (params) {
      const double ex = (m0 * px - m1 * py + m2 - qx) * g.isx, ey = (m1 * px + m0 * py + m3 - qy) * g.isy;
      w = recip_ge1(1.0 + (ex * ex + ey * ey) * g.inv_c2);
    }
    v[0] += w;
    v[1] += w * px;
    v[2] += w * py;
    v[3] += w * (px * px + py * py);
    v[4] += w * (px * qx + py * qy);
    v[5] += w * (px * qy - py * qx);
    v[6] += w * qx;
    v[7] += w * qy;
  }
#pragma unroll
  for (int k = 0; k < kGmSums; ++k) red[k][threadIdx.x] = v[k];
  gm_block_sum(red);
  if (threadIdx.x < kGmSums) partials[((size_t)b * gridDim.x + blockIdx.x) * kGmSums + threadIdx.x] = red[threadIdx.x][0];
}

// One block per pair: thread t adds partials t, t + 256, ... in order, then the fixed tree; thread 0 solves the normal
// equations of the similarity in closed form.  Round 0 records the weight fraction and flags a pair below the floor;
// a flagged pair keeps the identity through the later rounds.
__global__ void __launch_bounds__(kGmThreads) global_motion_pair_kernel(const double* __restrict__ partials, int chunks,
                                                                        int round, double npix, double min_weight,
                                                                        double* __restrict__ params,
                                                                        double* __restrict__ weight,
                                                                        uint8_t* __restrict__ flags,
                                                                        double* __restrict__ sums) {
  __shared__ double red[kGmSums][kGmThreads];
  const int b = blockIdx.x;
  const double* src = partials + (size_t)b * chunks * kGmSums;
  double v[kGmSums];
#pragma unroll
  for (int k = 0; k < kGmSums; ++k) v[k] = 0.0;
  for (int c = threadIdx.x; c < chunks; c += kGmThreads) {
#pragma unroll
    for (int k = 0; k < kGmSums; ++k) v[k] += src[(size_t)c * kGmSums + k];
  }
#pragma unroll
  for (int k = 0; k < kGmSums; ++k) red[k][threadIdx.x] = v[k];
  gm_block_sum(red);
  if (threadIdx.x != 0) return;
  const double S = red[0][0], X = red[1][0], Y = red[2][0], P = red[3][0], U = red[4][0], V = red[5][0],
               Qx = red[6][0], Qy = red[7][0];
  if (sums) {
#pragma unroll
    for (int k = 0; k < kGmSums; ++k) sums[(size_t)b * kGmSums + k] = red[k][0];
  }
  uint8_t flag = round == 0 ? 0 : flags[b];
  if (round == 0) {
    const double frac = S / npix;
    weight[b] = frac;
    flag = !(frac >= min_weight);
  }
  double a = 1.0, bb = 0.0, tx = 0.0, ty = 0.0;
  if (!flag) {
    const double den = P * S - X * X - Y * Y;
    if (!(S > 0.0) || !(den > kGmSingular * P * S)) {
      flag = 1;
    } else {
      a = (U * S - X * Qx - Y * Qy) / den;
      bb = (V * S - X * Qy + Y * Qx) / den;
      tx = (Qx - a * X + bb * Y) / S;
      ty = (Qy - bb * X - a * Y) / S;
      if (!(isfinite(a) && isfinite(bb) && isfinite(tx) && isfinite(ty))) {
        flag = 1;
        a = 1.0;
        bb = tx = ty = 0.0;
      }
    }
  }
  params[(size_t)b * 4 + 0] = a;
  params[(size_t)b * 4 + 1] = bb;
  params[(size_t)b * 4 + 2] = tx;
  params[(size_t)b * 4 + 3] = ty;
  flags[b] = flag;
}

static size_t global_motion_chunks(int Hn, int Wn) { return ((size_t)Hn * Wn + kGmChunk - 1) / kGmChunk; }

// One thread per output pixel of one frame; the source position in fp64 with every operation rounded on its own, rounded
// once to fp32, clamped into the frame (the border replicates) and sampled with the shared bilinear taps.
__global__ void __launch_bounds__(256) frames_warp_affine_kernel(const uint8_t* __restrict__ frames,
                                                                 const double* __restrict__ A, int H, int W, int C,
                                                                 uint8_t* __restrict__ out) {
  const size_t npix = (size_t)H * W;
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= npix) return;
  const int f = blockIdx.y;
  const double* m = A + (size_t)f * 6;
  const double x = (double)(q % (size_t)W), y = (double)(q / (size_t)W);
  const double sx = __dadd_rn(__dadd_rn(__dmul_rn(m[0], x), __dmul_rn(m[1], y)), m[2]);
  const double sy = __dadd_rn(__dadd_rn(__dmul_rn(m[3], x), __dmul_rn(m[4], y)), m[5]);
  // fmaxf(NaN, 0) = 0: a NaN position reads the top-left pixel rather than outside the frame
  const float fx = fminf(fmaxf(__double2float_rn(sx), 0.f), (float)(W - 1));
  const float fy = fminf(fmaxf(__double2float_rn(sy), 0.f), (float)(H - 1));
  const Bilerp bl = bilerp_at(fx, fy, H, W);
  const uint8_t* img = frames + (size_t)f * npix * C;
  const size_t i00 = ((size_t)bl.y0 * W + bl.x0) * C, i01 = ((size_t)bl.y0 * W + bl.x1) * C;
  const size_t i10 = ((size_t)bl.y1 * W + bl.x0) * C, i11 = ((size_t)bl.y1 * W + bl.x1) * C;
  uint8_t* dst = out + ((size_t)f * npix + q) * C;
  for (int c = 0; c < C; ++c) {
    const float v = bilerp1(bl, (float)img[i00 + c], (float)img[i01 + c], (float)img[i10 + c], (float)img[i11 + c]);
    dst[c] = (uint8_t)fminf(fmaxf(rintf(v), 0.f), 255.f);
  }
}

}  // namespace rb

using namespace rb;

extern "C" int rb_global_motion_workspace_bytes(int B, int Hn, int Wn, size_t* bytes) {
  RB_REQUIRE(bytes, RB_ERR_BAD_ARG, "rb_global_motion_workspace_bytes: null pointer");
  RB_REQUIRE(B > 0 && Hn > 0 && Wn > 0, RB_ERR_BAD_SHAPE, "rb_global_motion_workspace_bytes: bad shape B=%d Hn=%d Wn=%d",
             B, Hn, Wn);
  *bytes = (size_t)B * global_motion_chunks(Hn, Wn) * kGmSums * sizeof(double);
  return RB_OK;
}

extern "C" int rb_global_motion(const float* flow_fw, const uint8_t* occ_fw, int B, int Hn, int Wn, int Hs, int Ws,
                                float flow_scale, int rounds, double cauchy_c, double min_weight, double* params,
                                double* weight, uint8_t* flags, double* sums, void* workspace, size_t workspace_bytes,
                                void* stream) {
  RB_REQUIRE(flow_fw && occ_fw && params && weight && flags && workspace, RB_ERR_BAD_ARG,
             "rb_global_motion: null pointer");
  RB_REQUIRE(B > 0 && Hn > 0 && Wn > 0 && Hs > 0 && Ws > 0, RB_ERR_BAD_SHAPE,
             "rb_global_motion: bad shape B=%d Hn=%d Wn=%d Hs=%d Ws=%d", B, Hn, Wn, Hs, Ws);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "rb_global_motion: flow_scale must be finite and > 0 (got %g)", (double)flow_scale);
  RB_REQUIRE(rounds >= 0 && rounds <= RB_MOTION_MAX_ROUNDS, RB_ERR_BAD_ARG,
             "rb_global_motion: rounds must be in [0, %d] (got %d)", RB_MOTION_MAX_ROUNDS, rounds);
  RB_REQUIRE(cauchy_c > 0.0 && isfinite(cauchy_c), RB_ERR_BAD_ARG,
             "rb_global_motion: cauchy_c must be finite and > 0 (got %g)", cauchy_c);
  RB_REQUIRE(min_weight >= 0.0 && min_weight <= 1.0, RB_ERR_BAD_ARG,
             "rb_global_motion: min_weight must be in [0, 1] (got %g)", min_weight);
  const size_t npix = (size_t)Hn * Wn;
  const size_t chunks = global_motion_chunks(Hn, Wn);
  RB_REQUIRE(B <= 65535 && npix < (1ull << 31), RB_ERR_BAD_SHAPE,
             "rb_global_motion: B=%d pairs of %zu pixels exceed one grid", B, npix);
  const size_t need = (size_t)B * chunks * kGmSums * sizeof(double);
  RB_REQUIRE(workspace_bytes >= need, RB_ERR_WORKSPACE, "rb_global_motion: workspace of %zu bytes, %zu needed",
             workspace_bytes, need);
  GmGeom g;
  g.sx = (double)Ws / (double)Wn;
  g.sy = (double)Hs / (double)Hn;
  g.cx = 0.5 * (double)(Ws - 1);
  g.cy = 0.5 * (double)(Hs - 1);
  g.isx = (double)Wn / (double)Ws;
  g.isy = (double)Hn / (double)Hs;
  g.fs = (double)flow_scale;
  g.inv_c2 = 1.0 / (cauchy_c * cauchy_c);
  const cudaStream_t st = (cudaStream_t)stream;
  double* partials = static_cast<double*>(workspace);
  for (int r = 0; r <= rounds; ++r) {
    global_motion_chunk_kernel<<<dim3((unsigned)chunks, (unsigned)B), kGmThreads, 0, st>>>(
        reinterpret_cast<const float2*>(flow_fw), occ_fw, Wn, npix, g, r == 0 ? nullptr : params, partials);
    RB_CHECK_LAUNCH("global_motion_chunk_kernel");
    global_motion_pair_kernel<<<B, kGmThreads, 0, st>>>(partials, (int)chunks, r, (double)npix, min_weight, params,
                                                        weight, flags, r == rounds ? sums : nullptr);
    RB_CHECK_LAUNCH("global_motion_pair_kernel");
  }
  return RB_OK;
}

extern "C" int rb_frames_warp_affine(const uint8_t* frames, const double* A, int F, int H, int W, int C, uint8_t* out,
                                     void* stream) {
  RB_REQUIRE(frames && A && out, RB_ERR_BAD_ARG, "rb_frames_warp_affine: null pointer");
  RB_REQUIRE(F > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_frames_warp_affine: bad shape F=%d H=%d W=%d", F, H, W);
  RB_REQUIRE(C >= 1 && C <= 4, RB_ERR_BAD_ARG, "rb_frames_warp_affine: C must be in [1, 4] (got %d)", C);
  const size_t npix = (size_t)H * W;
  const size_t blocks = (npix + 255) / 256;
  RB_REQUIRE(F <= 65535 && blocks <= 0x7fffffffu && W < (1 << 24) && H < (1 << 24), RB_ERR_BAD_SHAPE,
             "rb_frames_warp_affine: F=%d frames of %dx%d pixels exceed one grid", F, H, W);
  RB_REQUIRE(frames != out, RB_ERR_BAD_ARG, "rb_frames_warp_affine: out must not alias frames");
  frames_warp_affine_kernel<<<dim3((unsigned)blocks, (unsigned)F), 256, 0, (cudaStream_t)stream>>>(frames, A, H, W, C,
                                                                                                  out);
  RB_CHECK_LAUNCH("frames_warp_affine_kernel");
  return RB_OK;
}
