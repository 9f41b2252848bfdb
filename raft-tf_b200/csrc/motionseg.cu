// F34 / F35: motion segmentation -- a robust homography fit of each frame pair's camera motion to its flow
// (rb_homography_motion), the per-pixel evidence of motion that departs from it (rb_motion_evidence), and its aggregation
// along the chained flow of neighbouring frames into a binary mask per frame pixel (rb_motion_segment).  The fit reduces
// in fp64 in a fixed order; the evidence and the segmentation round every operation on its own (__dadd_rn / __fmul_rn /
// ..., no FMA contraction), so a numpy restatement reproduces their bits (tests/motionseg_oracle.py).  No atomics.
#include <math.h>

#include <algorithm>

#include "common.cuh"
#include "fb_sample.cuh"

namespace rb {

constexpr int kHmThreads = 256;
constexpr int kHmWarps = kHmThreads / 32;
constexpr int kHmPerThread = 16;
constexpr int kHmChunk = kHmThreads * kHmPerThread;  // pixels per block, as F22
constexpr int kHmSums = RB_HOMOGRAPHY_SUMS;           // S, 36 of the upper triangle of the 8 x 8 system, 8 of its rhs
constexpr double kHmSingular = 1e-12;                 // a Cholesky pivot at or below this fraction of its diagonal
constexpr int kSegThreads = 256;

// The frames' geometry as F22's GmGeom, plus the normalisation: a centred point p is (x, y) = p / L, L = max(Ws, Hs) / 2.
struct HmGeom {
  double sx, sy, cx, cy, isx, isy, fs, inv_c2, L, invL;
};

// index of entry (i, j), i <= j, of the 8 x 8 system's upper triangle in the sums (after S), row by row
__host__ __device__ constexpr int hm_tri(int i, int j) { return 1 + i * 8 - i * (i - 1) / 2 + (j - i); }

// Fixed-shape sum of all 45 values over the block: a shuffle tree per warp (lane offsets 16, 8, 4, 2, 1), then the 8 warp
// totals in warp order by threads 0..44 into out.
__device__ __forceinline__ void hm_block_sum(double (&v)[kHmSums], double (*red)[kHmWarps], double* out) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < kHmSums; ++k) {
    double s = v[k];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
    if (lane == 0) red[k][wid] = s;
  }
  __syncthreads();
  if (threadIdx.x < kHmSums) {
    double s = red[threadIdx.x][0];
#pragma unroll
    for (int w = 1; w < kHmWarps; ++w) s += red[threadIdx.x][w];
    out[threadIdx.x] = s;
  }
}

// 1 / d for a finite d > 0 to within an ulp: the hardware's approximate fp64 reciprocal refined by two Newton steps (the
// correctly rounded division calls a slow path that makes ptxas spill in the pixel loop)
__device__ __forceinline__ double hm_recip(double d) {
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(d));
  y = fma(y, fma(-d, y, 1.0), y);
  return fma(y, fma(-d, y, 1.0), y);
}

// Round 0's previous estimate: the similarity (a, b, tx, ty) of F22 in normalised coordinates, or the identity with flag 2
// for a pair F22 flagged.
__global__ void homography_init_kernel(const double* __restrict__ sim, const uint8_t* __restrict__ sim_flags, int B,
                                       double invL, double* __restrict__ H, uint8_t* __restrict__ flags) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  double* h = H + (size_t)b * 9;
  const bool bad = sim_flags[b] != 0;
  const double a = bad ? 1.0 : sim[(size_t)b * 4], s = bad ? 0.0 : sim[(size_t)b * 4 + 1];
  const double tx = bad ? 0.0 : sim[(size_t)b * 4 + 2] * invL, ty = bad ? 0.0 : sim[(size_t)b * 4 + 3] * invL;
  h[0] = a, h[1] = -s, h[2] = tx, h[3] = s, h[4] = a, h[5] = ty, h[6] = 0.0, h[7] = 0.0, h[8] = 1.0;
  flags[b] = bad ? 2 : 0;
}

// grid (chunks per pair, B); thread t takes pixels chunk_start + k * 256 + t, k = 0..15 in order (coalesced).  A pixel with
// occ == 0 and a finite flow weighs the Cauchy weight of its residual under the previous estimate H, over z^2.
__global__ void __launch_bounds__(kHmThreads) homography_chunk_kernel(const float2* __restrict__ flow,
                                                                      const uint8_t* __restrict__ occ, int Wn, size_t npix,
                                                                      HmGeom g, const double* __restrict__ H,
                                                                      double* __restrict__ partials) {
  __shared__ double red[kHmSums][kHmWarps];
  const int b = blockIdx.y;
  const size_t base = (size_t)b * npix;
  const size_t c0 = (size_t)blockIdx.x * kHmChunk;
  double h[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) h[k] = H[(size_t)b * 9 + k];
  double v[kHmSums];
#pragma unroll
  for (int k = 0; k < kHmSums; ++k) v[k] = 0.0;
  for (int k = 0; k < kHmPerThread; ++k) {
    const size_t q = c0 + (size_t)k * kHmThreads + threadIdx.x;
    if (q >= npix) break;
    const size_t p = base + q;
    const float2 f = flow[p];
    if (occ[p] != 0 || !isfinite(f.x) || !isfinite(f.y)) continue;
    const int i = (int)q / Wn, j = (int)q % Wn;  // npix < 2^31
    const double px = ((double)j + 0.5) * g.sx - 0.5 - g.cx, py = ((double)i + 0.5) * g.sy - 0.5 - g.cy;
    const double x = px * g.invL, y = py * g.invL;
    const double ux = (px + g.fs * ((double)f.x * g.sx)) * g.invL, uy = (py + g.fs * ((double)f.y * g.sy)) * g.invL;
    const double z = h[6] * x + h[7] * y + 1.0;
    if (!(z > 0.0)) continue;
    const double iz = hm_recip(z);
    const double ex = ((h[0] * x + h[1] * y + h[2]) * iz - ux) * (g.L * g.isx);
    const double ey = ((h[3] * x + h[4] * y + h[5]) * iz - uy) * (g.L * g.isy);
    const double r2 = ex * ex + ey * ey;
    if (!isfinite(r2)) continue;
    const double w = hm_recip(1.0 + r2 * g.inv_c2) * (iz * iz);
    const double ax[8] = {x, y, 1.0, 0.0, 0.0, 0.0, -x * ux, -y * ux};
    const double ay[8] = {0.0, 0.0, 0.0, x, y, 1.0, -x * uy, -y * uy};
    v[0] += w;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
#pragma unroll
      for (int c = r; c < 8; ++c) v[hm_tri(r, c)] += w * (ax[r] * ax[c] + ay[r] * ay[c]);
      v[37 + r] += w * (ax[r] * ux + ay[r] * uy);
    }
  }
  hm_block_sum(v, red, partials + ((size_t)b * gridDim.x + blockIdx.x) * kHmSums);
}

// One block per pair: thread t adds partials t, t + 256, ... in order, then the fixed block sum; thread 0 solves the
// normal equations by Cholesky in fp64.  A pair already flagged keeps its H; a singular round flags it 1 and restores the
// initial similarity.
__global__ void __launch_bounds__(kHmThreads) homography_pair_kernel(const double* __restrict__ partials, int chunks,
                                                                     const double* __restrict__ sim, double invL,
                                                                     double* __restrict__ H,
                                                                     uint8_t* __restrict__ flags,
                                                                     double* __restrict__ sums) {
  __shared__ double red[kHmSums][kHmWarps];
  __shared__ double tot[kHmSums];
  const int b = blockIdx.x;
  const double* src = partials + (size_t)b * chunks * kHmSums;
  double v[kHmSums];
#pragma unroll
  for (int k = 0; k < kHmSums; ++k) v[k] = 0.0;
  for (int c = threadIdx.x; c < chunks; c += kHmThreads) {
#pragma unroll
    for (int k = 0; k < kHmSums; ++k) v[k] += src[(size_t)c * kHmSums + k];
  }
  hm_block_sum(v, red, tot);
  __syncthreads();
  if (threadIdx.x != 0) return;
  if (sums) {
    for (int k = 0; k < kHmSums; ++k) sums[(size_t)b * kHmSums + k] = tot[k];
  }
  if (flags[b] != 0) return;
  // A = L L^T in place (lower triangle), then L y = rhs, L^T h = y
  double A[8][8], y[8];
  for (int r = 0; r < 8; ++r)
    for (int c = r; c < 8; ++c) A[c][r] = tot[hm_tri(r, c)];
  bool ok = tot[0] > 0.0;
  for (int j = 0; j < 8 && ok; ++j) {
    double d = A[j][j];
    for (int k = 0; k < j; ++k) d -= A[j][k] * A[j][k];
    if (!(d > kHmSingular * A[j][j])) {
      ok = false;
      break;
    }
    const double l = sqrt(d);
    A[j][j] = l;
    for (int i = j + 1; i < 8; ++i) {
      double s = A[i][j];
      for (int k = 0; k < j; ++k) s -= A[i][k] * A[j][k];
      A[i][j] = s / l;
    }
  }
  double hn[8];
  if (ok) {
    for (int i = 0; i < 8; ++i) {
      double s = tot[37 + i];
      for (int k = 0; k < i; ++k) s -= A[i][k] * y[k];
      y[i] = s / A[i][i];
    }
    for (int i = 7; i >= 0; --i) {
      double s = y[i];
      for (int k = i + 1; k < 8; ++k) s -= A[k][i] * hn[k];
      hn[i] = s / A[i][i];
      ok = ok && isfinite(hn[i]);
    }
  }
  double* h = H + (size_t)b * 9;
  if (ok) {
    for (int k = 0; k < 8; ++k) h[k] = hn[k];
  } else {
    const double a = sim[(size_t)b * 4], s = sim[(size_t)b * 4 + 1];
    h[0] = a, h[1] = -s, h[2] = sim[(size_t)b * 4 + 2] * invL, h[3] = s, h[4] = a, h[5] = sim[(size_t)b * 4 + 3] * invL;
    h[6] = 0.0, h[7] = 0.0;
    flags[b] = 1;
  }
  h[8] = 1.0;
}

static size_t homography_chunks(int Hn, int Wn) { return ((size_t)Hn * Wn + kHmChunk - 1) / kHmChunk; }

// e = r^2 / (r^2 + tau^2) of one field at network pixel (i, j): r the residual of p's flow target against H p in network
// pixels, in fp64 with every operation rounded on its own, r^2 rounded once to fp32; 1 where H p is behind the camera or
// r^2 is not finite.
__device__ __forceinline__ float motion_e(float2 f, int i, int j, const double* __restrict__ h, const HmGeom& g,
                                          float tau2) {
  const double px = __dsub_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)j, 0.5), g.sx), 0.5), g.cx);
  const double py = __dsub_rn(__dsub_rn(__dmul_rn(__dadd_rn((double)i, 0.5), g.sy), 0.5), g.cy);
  const double x = __dmul_rn(px, g.invL), y = __dmul_rn(py, g.invL);
  const double ux = __dmul_rn(__dadd_rn(px, __dmul_rn(g.fs, __dmul_rn((double)f.x, g.sx))), g.invL);
  const double uy = __dmul_rn(__dadd_rn(py, __dmul_rn(g.fs, __dmul_rn((double)f.y, g.sy))), g.invL);
  const double z = __dadd_rn(__dadd_rn(__dmul_rn(h[6], x), __dmul_rn(h[7], y)), 1.0);
  if (!(z > 0.0)) return 1.f;
  const double X = __dadd_rn(__dadd_rn(__dmul_rn(h[0], x), __dmul_rn(h[1], y)), h[2]);
  const double Y = __dadd_rn(__dadd_rn(__dmul_rn(h[3], x), __dmul_rn(h[4], y)), h[5]);
  const double dx = __dmul_rn(__dmul_rn(__dsub_rn(__ddiv_rn(X, z), ux), g.L), g.isx);
  const double dy = __dmul_rn(__dmul_rn(__dsub_rn(__ddiv_rn(Y, z), uy), g.L), g.isy);
  const float r2 = __double2float_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)));
  if (!isfinite(r2)) return 1.f;
  return __fdiv_rn(r2, __fadd_rn(r2, tau2));
}

// One thread per network pixel of frame t (blockIdx.y): (N, C) from +0, the forward field of pair t, then the backward
// field of pair t - 1, each where it is consistent, finite, fitted (flag <= 1) and not a cut pair.
__global__ void __launch_bounds__(256) motion_evidence_kernel(const float2* __restrict__ fw, const float2* __restrict__ bw,
                                                              const uint8_t* __restrict__ occ_fw,
                                                              const uint8_t* __restrict__ occ_bw,
                                                              const double* __restrict__ H,
                                                              const uint8_t* __restrict__ flags,
                                                              const uint8_t* __restrict__ cuts, int T, int Wn,
                                                              size_t npix, HmGeom g, float tau2,
                                                              float2* __restrict__ ev) {
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= npix) return;
  const int t = blockIdx.y;
  const int i = (int)(q / (size_t)Wn), j = (int)(q % (size_t)Wn);
  float N = 0.f, C = 0.f;
#pragma unroll
  for (int side = 0; side < 2; ++side) {
    const int k = side == 0 ? t : t - 1;  // the pair
    if (k < 0 || k >= T) continue;
    const int field = side == 0 ? k : T + k;
    if (flags[field] > 1 || (cuts && cuts[k])) continue;
    const size_t p = (size_t)k * npix + q;
    const float2 f = side == 0 ? fw[p] : bw[p];
    if ((side == 0 ? occ_fw[p] : occ_bw[p]) != 0 || !isfinite(f.x) || !isfinite(f.y)) continue;
    N = __fadd_rn(N, motion_e(f, i, j, H + (size_t)field * 9, g, tau2));
    C = __fadd_rn(C, 1.f);
  }
  ev[(size_t)t * npix + q] = make_float2(N, C);
}

// (N, C) of evidence map ev [Hn,Wn] sampled bilinearly at the taps of b
__device__ __forceinline__ float2 sample_ev(const float2* __restrict__ ev, int Wn, const Bilerp& b) {
  const float2 v00 = ev[(size_t)b.y0 * Wn + b.x0], v01 = ev[(size_t)b.y0 * Wn + b.x1];
  const float2 v10 = ev[(size_t)b.y1 * Wn + b.x0], v11 = ev[(size_t)b.y1 * Wn + b.x1];
  return make_float2(bilerp1(b, v00.x, v01.x, v10.x, v11.x), bilerp1(b, v00.y, v01.y, v10.y, v11.y));
}

// One thread per frame pixel, blockIdx.y over the rows (striding); row r = (t, nf, nb).  Each side chains steps until
// one leaves the grid or fails the F5 test, as rb_denoise_merge's sides do.
__global__ void __launch_bounds__(kSegThreads) motion_segment_kernel(const float2* __restrict__ ev, int F, int Hn, int Wn,
                                                                     const float2* __restrict__ fw,
                                                                     const float2* __restrict__ bw, int Hs, int Ws,
                                                                     NetGeom g, float s, float a1, float a2,
                                                                     const int32_t* __restrict__ rows, int n_rows,
                                                                     uint8_t* __restrict__ mask,
                                                                     uint8_t* __restrict__ status) {
  const size_t ns = (size_t)Hs * Ws, nn = (size_t)Hn * Wn;
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= ns) return;
  const int x = (int)(q % Ws), y = (int)(q / Ws);
  for (int r = blockIdx.y; r < n_rows; r += gridDim.y) {
    const int t = __ldg(rows + 3 * r), nf = __ldg(rows + 3 * r + 1), nb = __ldg(rows + 3 * r + 2);
    const size_t o = (size_t)r * ns + q;
    if (t < 0 || t >= F) {  // an absent row
      mask[o] = 0;
      status[o] = 1;
      continue;
    }
    const float2 p0 = make_float2(px_remap(x, g.rxn, Wn), px_remap(y, g.ryn, Hn));
    float2 acc = sample_ev(ev + (size_t)t * nn, Wn, bilerp_at(p0.x, p0.y, Hn, Wn));
#pragma unroll 1
    for (int dir = 1; dir >= -1; dir -= 2) {
      const int n = dir > 0 ? min(min(max(nf, 0), RB_MOTION_SEG_MAX_WINDOW), F - 1 - t)
                            : min(min(max(nb, 0), RB_MOTION_SEG_MAX_WINDOW), t);
      float2 p = p0;
      for (int step = 1; step <= n; ++step) {
        const ChainLink l = chain_link(fw, bw, nn, t, dir, step);
        float2 qq;
        if (chain_step(l.pull, l.test, Hn, Wn, s, a1, a2, p, qq)) break;
        p = qq;
        const float2 e = sample_ev(ev + (size_t)(t + dir * step) * nn, Wn, bilerp_at(p.x, p.y, Hn, Wn));
        acc = make_float2(__fadd_rn(acc.x, e.x), __fadd_rn(acc.y, e.y));
      }
    }
    mask[o] = acc.y > 0.f && __fmul_rn(2.f, acc.x) >= acc.y ? 1 : 0;
    status[o] = acc.y > 0.f ? 0 : 1;
  }
}

static HmGeom hm_geom(int Hn, int Wn, int Hs, int Ws, float flow_scale, double cauchy_c) {
  HmGeom g;
  g.sx = (double)Ws / (double)Wn;
  g.sy = (double)Hs / (double)Hn;
  g.cx = 0.5 * (double)(Ws - 1);
  g.cy = 0.5 * (double)(Hs - 1);
  g.isx = (double)Wn / (double)Ws;
  g.isy = (double)Hn / (double)Hs;
  g.fs = (double)flow_scale;
  g.inv_c2 = 1.0 / (cauchy_c * cauchy_c);
  g.L = 0.5 * (double)std::max(Ws, Hs);
  g.invL = 1.0 / g.L;
  return g;
}

}  // namespace rb

using namespace rb;

extern "C" int rb_homography_motion_workspace_bytes(int B, int Hn, int Wn, size_t* bytes) {
  RB_REQUIRE(bytes, RB_ERR_BAD_ARG, "rb_homography_motion_workspace_bytes: null pointer");
  RB_REQUIRE(B > 0 && Hn > 0 && Wn > 0, RB_ERR_BAD_SHAPE,
             "rb_homography_motion_workspace_bytes: bad shape B=%d Hn=%d Wn=%d", B, Hn, Wn);
  *bytes = (size_t)B * homography_chunks(Hn, Wn) * kHmSums * sizeof(double);
  return RB_OK;
}

extern "C" int rb_homography_motion(const float* flow, const uint8_t* occ, int B, int Hn, int Wn, int Hs, int Ws,
                                    float flow_scale, const double* sim_params, const uint8_t* sim_flags, int rounds,
                                    double cauchy_c, double* H, uint8_t* flags, double* sums, void* workspace,
                                    size_t workspace_bytes, void* stream) {
  RB_REQUIRE(flow && occ && sim_params && sim_flags && H && flags && workspace, RB_ERR_BAD_ARG,
             "rb_homography_motion: null pointer");
  RB_REQUIRE(B > 0 && Hn > 0 && Wn > 0 && Hs > 0 && Ws > 0, RB_ERR_BAD_SHAPE,
             "rb_homography_motion: bad shape B=%d Hn=%d Wn=%d Hs=%d Ws=%d", B, Hn, Wn, Hs, Ws);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "rb_homography_motion: flow_scale must be finite and > 0 (got %g)", (double)flow_scale);
  RB_REQUIRE(rounds >= 1 && rounds <= RB_HOMOGRAPHY_MAX_ROUNDS, RB_ERR_BAD_ARG,
             "rb_homography_motion: rounds must be in [1, %d] (got %d)", RB_HOMOGRAPHY_MAX_ROUNDS, rounds);
  RB_REQUIRE(cauchy_c > 0.0 && isfinite(cauchy_c), RB_ERR_BAD_ARG,
             "rb_homography_motion: cauchy_c must be finite and > 0 (got %g)", cauchy_c);
  const size_t npix = (size_t)Hn * Wn;
  const size_t chunks = homography_chunks(Hn, Wn);
  RB_REQUIRE(B <= 65535 && npix < (1ull << 31), RB_ERR_BAD_SHAPE,
             "rb_homography_motion: B=%d pairs of %zu pixels exceed one grid", B, npix);
  const size_t need = (size_t)B * chunks * kHmSums * sizeof(double);
  RB_REQUIRE(workspace_bytes >= need, RB_ERR_WORKSPACE, "rb_homography_motion: workspace of %zu bytes, %zu needed",
             workspace_bytes, need);
  const HmGeom g = hm_geom(Hn, Wn, Hs, Ws, flow_scale, cauchy_c);
  const cudaStream_t st = (cudaStream_t)stream;
  double* partials = static_cast<double*>(workspace);
  homography_init_kernel<<<(B + 127) / 128, 128, 0, st>>>(sim_params, sim_flags, B, g.invL, H, flags);
  RB_CHECK_LAUNCH("homography_init_kernel");
  for (int r = 0; r < rounds; ++r) {
    homography_chunk_kernel<<<dim3((unsigned)chunks, (unsigned)B), kHmThreads, 0, st>>>(
        reinterpret_cast<const float2*>(flow), occ, Wn, npix, g, H, partials);
    RB_CHECK_LAUNCH("homography_chunk_kernel");
    homography_pair_kernel<<<B, kHmThreads, 0, st>>>(partials, (int)chunks, sim_params, g.invL, H, flags,
                                                     r == rounds - 1 ? sums : nullptr);
    RB_CHECK_LAUNCH("homography_pair_kernel");
  }
  return RB_OK;
}

extern "C" int rb_motion_evidence(const float* flow_fw, const float* flow_bw, const uint8_t* occ_fw,
                                  const uint8_t* occ_bw, const double* H, const uint8_t* flags, const uint8_t* cuts,
                                  int T, int Hn, int Wn, int Hs, int Ws, float flow_scale, float tau, float* evidence,
                                  void* stream) {
  RB_REQUIRE(flow_fw && flow_bw && occ_fw && occ_bw && H && flags && evidence, RB_ERR_BAD_ARG,
             "rb_motion_evidence: null pointer");
  RB_REQUIRE(T > 0 && Hn > 0 && Wn > 0 && Hs > 0 && Ws > 0, RB_ERR_BAD_SHAPE,
             "rb_motion_evidence: bad shape T=%d Hn=%d Wn=%d Hs=%d Ws=%d", T, Hn, Wn, Hs, Ws);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "rb_motion_evidence: flow_scale must be finite and > 0 (got %g)", (double)flow_scale);
  RB_REQUIRE(tau > 0.f && isfinite(tau), RB_ERR_BAD_ARG, "rb_motion_evidence: tau must be finite and > 0 (got %g)",
             (double)tau);
  const size_t npix = (size_t)Hn * Wn;
  const size_t blocks = (npix + 255) / 256;
  RB_REQUIRE(T < 65535 && npix < (1ull << 31), RB_ERR_BAD_SHAPE,
             "rb_motion_evidence: %d frames of %zu pixels exceed one grid", T + 1, npix);
  const HmGeom g = hm_geom(Hn, Wn, Hs, Ws, flow_scale, 1.0);
  motion_evidence_kernel<<<dim3((unsigned)blocks, (unsigned)(T + 1)), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw), occ_fw, occ_bw, H, flags, cuts,
      T, Wn, npix, g, tau * tau, reinterpret_cast<float2*>(evidence));
  RB_CHECK_LAUNCH("motion_evidence_kernel");
  return RB_OK;
}

extern "C" int rb_motion_segment(const float* evidence, int F, int Hn, int Wn, const float* flow_fw,
                                 const float* flow_bw, int Hs, int Ws, float flow_scale, float alpha1, float alpha2,
                                 const int32_t* rows, int n_rows, uint8_t* mask, uint8_t* status, void* stream) {
  const char* fn = "rb_motion_segment";
  if (int rc = check_rows_entry(fn, evidence && rows && mask && status, flow_fw, flow_bw, F, Hs, Ws, Hn, Wn, n_rows))
    return rc;
  if (int rc = check_rows_step(fn, Hs, Ws, flow_scale, alpha1, alpha2)) return rc;
  motion_segment_kernel<<<rows_grid(Hs, Ws, kSegThreads, n_rows), kSegThreads, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float2*>(evidence), F, Hn, Wn, reinterpret_cast<const float2*>(flow_fw),
      reinterpret_cast<const float2*>(flow_bw), Hs, Ws, net_geom(Hs, Ws, Hn, Wn), flow_scale, alpha1, alpha2, rows,
      n_rows, mask, status);
  RB_CHECK_LAUNCH("motion_segment_kernel");
  return RB_OK;
}
