// F24 / F25: object removal from video -- the membrane fill of a field inside a hole (flow completion and the spatial
// fill), the hole masks at the frames' size and on the network grid, and the temporal fill that follows the completed
// flows to the nearest frames that see behind the hole.  Every fp32 operation is rounded on its own (__fadd_rn /
// __fmul_rn / __fsub_rn / __fdiv_rn, no FMA contraction), so a numpy restatement reproduces the bits
// (tests/inpaint_oracle.py); no atomics.
#include <math.h>

#include "common.cuh"
#include "fb_sample.cuh"

namespace rb {

constexpr int kFillMaxLevels = 32;
constexpr int kFillSmall = 4096;  // levels of at most this many pixels run their part of a V-cycle in one CTA per field
constexpr int kFillThreads = 256;
constexpr int kFillSmallThreads = 1024;

// One pyramid level of all B fields: values (level 0: the caller's field; coarser: the initial guess, then the
// correction), right-hand side (coarser levels only) and mask.  Level 0's mask is the caller's hole map (non-zero =
// hole); a coarser level's has bit 0 set when no child is known (a hole of the initial guess) and bit 1 when every child
// is a hole of the finer level's correction problem.
struct FillLevel {
  float* v;
  float* f;
  uint8_t* m;
  int h, w;
};

struct FillPyr {
  FillLevel l[kFillMaxLevels];
  int L;
  const float* lohi;  // [B][2][C]: the smallest and largest known value of each channel (0, 0 without any)
};

enum FillOp { kRestrictInit, kProlongInit, kDirichlet, kCorrect, kResidualDown, kProlongAdd };

// Level lv of field b.
template <int C>
__device__ __forceinline__ FillLevel field_level(const FillPyr& P, int lv, int b) {
  FillLevel L = P.l[lv];
  const size_t hw = (size_t)L.h * L.w;
  L.v += (size_t)b * hw * C;
  if (L.f) L.f += (size_t)b * hw * C;
  L.m += (size_t)b * hw;
  return L;
}

__device__ __forceinline__ bool init_hole(const FillLevel& L, int lv, size_t q) {
  return lv == 0 ? L.m[q] != 0 : (L.m[q] & 1) != 0;
}
__device__ __forceinline__ bool corr_hole(const FillLevel& L, int lv, size_t q) {
  return lv == 0 ? L.m[q] != 0 : (L.m[q] & 2) != 0;
}

// The rounded mean of up to four values in order: s = 0 + v0 + v1 + ..., s / n, clamped by comparisons into the
// values' [min, max] -- so it never leaves the range of what it averages, and a constant stays bit for bit.
template <int C>
struct Mean {
  float s[C], lo[C], hi[C];
  int n = 0;
  __device__ __forceinline__ Mean() {
#pragma unroll
    for (int c = 0; c < C; ++c) s[c] = lo[c] = hi[c] = 0.f;
  }
  __device__ __forceinline__ void add(const float* v) {
#pragma unroll
    for (int c = 0; c < C; ++c) {
      if (n == 0 || v[c] < lo[c]) lo[c] = v[c];
      if (n == 0 || v[c] > hi[c]) hi[c] = v[c];
      s[c] = __fadd_rn(s[c], v[c]);
    }
    ++n;
  }
  __device__ __forceinline__ void store(float* out) const {
#pragma unroll
    for (int c = 0; c < C; ++c) {
      float m = __fdiv_rn(s[c], (float)n);
      if (m < lo[c]) m = lo[c];
      if (m > hi[c]) m = hi[c];
      out[c] = m;
    }
  }
};

// Coarse pixel q of level lv >= 1 from its <= 4 children in tap order (2i,2j), (2i,2j+1), (2i+1,2j), (2i+1,2j+1).
template <int C>
__device__ void restrict_init(const FillPyr& P, int lv, int b, size_t q) {
  const FillLevel F = field_level<C>(P, lv - 1, b), K = field_level<C>(P, lv, b);
  const int i = (int)(q / K.w), j = (int)(q % K.w);
  Mean<C> mean;
  bool all_corr = true;
  for (int t = 0; t < 4; ++t) {
    const int y = 2 * i + (t >> 1), x = 2 * j + (t & 1);
    if (y >= F.h || x >= F.w) continue;
    const size_t p = (size_t)y * F.w + x;
    all_corr = all_corr && corr_hole(F, lv - 1, p);
    if (!init_hole(F, lv - 1, p)) mean.add(F.v + p * C);
  }
  float out[C];
  if (mean.n) {
    mean.store(out);
  } else {
#pragma unroll
    for (int c = 0; c < C; ++c) out[c] = 0.f;
  }
#pragma unroll
  for (int c = 0; c < C; ++c) K.v[q * C + c] = out[c];
  K.m[q] = (uint8_t)((mean.n ? 0 : 1) | (all_corr ? 2 : 0));
}

// A hole pixel of the initial guess at level lv takes its parent's value (nearest).
template <int C>
__device__ void prolong_init(const FillPyr& P, int lv, int b, size_t q) {
  const FillLevel F = field_level<C>(P, lv, b);
  if (!init_hole(F, lv, q)) return;
  const FillLevel K = field_level<C>(P, lv + 1, b);
  const int i = (int)(q / F.w), j = (int)(q % F.w);
  const size_t p = (size_t)(i >> 1) * K.w + (j >> 1);
#pragma unroll
  for (int c = 0; c < C; ++c) F.v[q * C + c] = K.v[p * C + c];
}

// The in-image neighbours of pixel (i, j) in the order up, down, left, right.
__device__ __forceinline__ int neighbours(int i, int j, int h, int w, size_t* nb) {
  int n = 0;
  if (i > 0) nb[n++] = (size_t)(i - 1) * w + j;
  if (i + 1 < h) nb[n++] = (size_t)(i + 1) * w + j;
  if (j > 0) nb[n++] = (size_t)i * w + j - 1;
  if (j + 1 < w) nb[n++] = (size_t)i * w + j + 1;
  return n;
}

// One colour of a Gauss-Seidel sweep of the membrane equation (omega = 1): a hole pixel becomes the rounded mean of its
// neighbours.
template <int C>
__device__ void dirichlet(const FillPyr& P, int lv, int b, size_t q, int colour) {
  const FillLevel F = field_level<C>(P, lv, b);
  const int i = (int)(q / F.w), j = (int)(q % F.w);
  if (((i + j) & 1) != colour || !init_hole(F, lv, q)) return;
  size_t nb[4];
  const int n = neighbours(i, j, F.h, F.w, nb);
  if (!n) return;
  Mean<C> mean;
  for (int k = 0; k < n; ++k) mean.add(F.v + nb[k] * C);
  mean.store(F.v + q * C);
}

// s = f + the neighbours' values (each sum rounded, f = 0 on level 0), and their count.
template <int C>
__device__ __forceinline__ int neighbour_sum(const FillLevel& F, int lv, size_t q, float* s) {
  const int i = (int)(q / F.w), j = (int)(q % F.w);
#pragma unroll
  for (int c = 0; c < C; ++c) s[c] = lv == 0 ? 0.f : F.f[q * C + c];
  size_t nb[4];
  const int n = neighbours(i, j, F.h, F.w, nb);
  for (int k = 0; k < n; ++k) {
#pragma unroll
    for (int c = 0; c < C; ++c) s[c] = __fadd_rn(s[c], F.v[nb[k] * C + c]);
  }
  return n;
}

// One colour of a Gauss-Seidel sweep of the correction equation n e_p - sum e_nb = f_p (level lv >= 1).
template <int C>
__device__ void correct(const FillPyr& P, int lv, int b, size_t q, int colour) {
  const FillLevel F = field_level<C>(P, lv, b);
  const int i = (int)(q / F.w), j = (int)(q % F.w);
  if (((i + j) & 1) != colour || !corr_hole(F, lv, q)) return;
  float s[C];
  const int n = neighbour_sum<C>(F, lv, q, s);
  if (!n) return;
#pragma unroll
  for (int c = 0; c < C; ++c) F.v[q * C + c] = __fdiv_rn(s[c], (float)n);
}

// Coarse pixel q of level lv + 1: f = 0 + the residuals s - n v of its four children in tap order (0 for a child
// outside level lv or off its correction hole), and a zero correction.
template <int C>
__device__ void residual_down(const FillPyr& P, int lv, int b, size_t q) {
  const FillLevel F = field_level<C>(P, lv, b), K = field_level<C>(P, lv + 1, b);
  const int i = (int)(q / K.w), j = (int)(q % K.w);
  float out[C];
#pragma unroll
  for (int c = 0; c < C; ++c) out[c] = 0.f;
  for (int t = 0; t < 4; ++t) {
    const int y = 2 * i + (t >> 1), x = 2 * j + (t & 1);
    float r[C];
#pragma unroll
    for (int c = 0; c < C; ++c) r[c] = 0.f;
    if (y < F.h && x < F.w) {
      const size_t p = (size_t)y * F.w + x;
      if (corr_hole(F, lv, p)) {
        float s[C];
        const int n = neighbour_sum<C>(F, lv, p, s);
#pragma unroll
        for (int c = 0; c < C; ++c) r[c] = __fsub_rn(s[c], __fmul_rn((float)n, F.v[p * C + c]));
      }
    }
#pragma unroll
    for (int c = 0; c < C; ++c) out[c] = __fadd_rn(out[c], r[c]);
  }
#pragma unroll
  for (int c = 0; c < C; ++c) {
    K.f[q * C + c] = out[c];
    K.v[q * C + c] = 0.f;
  }
}

// The two coarse taps of fine index z and their weights: cell-centred bilinear, 1/4 and 3/4, clamped into n.
__device__ __forceinline__ void prolong_taps(int z, int n, int* a, int* bb, float* wa, float* wb) {
  const int i = z >> 1;
  if ((z & 1) == 0) {
    *a = max(i - 1, 0);
    *bb = i;
    *wa = 0.25f;
    *wb = 0.75f;
  } else {
    *a = i;
    *bb = min(i + 1, n - 1);
    *wa = 0.75f;
    *wb = 0.25f;
  }
}

// A correction-hole pixel of level lv adds the bilinear value of level lv + 1's correction; on level 0 the sum is
// clamped into the field's known range.
template <int C>
__device__ void prolong_add(const FillPyr& P, int lv, int b, size_t q) {
  const FillLevel F = field_level<C>(P, lv, b);
  if (!corr_hole(F, lv, q)) return;
  const FillLevel K = field_level<C>(P, lv + 1, b);
  const int i = (int)(q / F.w), j = (int)(q % F.w);
  int ya, yb, xa, xb;
  float wya, wyb, wxa, wxb;
  prolong_taps(i, K.h, &ya, &yb, &wya, &wyb);
  prolong_taps(j, K.w, &xa, &xb, &wxa, &wxb);
  const float* e = K.v;
  const size_t p00 = ((size_t)ya * K.w + xa) * C, p01 = ((size_t)ya * K.w + xb) * C;
  const size_t p10 = ((size_t)yb * K.w + xa) * C, p11 = ((size_t)yb * K.w + xb) * C;
  const float* lohi = P.lohi + (size_t)b * 2 * C;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const float t0 = __fadd_rn(__fmul_rn(wxa, e[p00 + c]), __fmul_rn(wxb, e[p01 + c]));
    const float t1 = __fadd_rn(__fmul_rn(wxa, e[p10 + c]), __fmul_rn(wxb, e[p11 + c]));
    float v = __fadd_rn(F.v[q * C + c], __fadd_rn(__fmul_rn(t0, wya), __fmul_rn(t1, wyb)));
    if (lv == 0) {
      if (v < lohi[c]) v = lohi[c];
      if (v > lohi[C + c]) v = lohi[C + c];
    }
    F.v[q * C + c] = v;
  }
}

template <int C>
__device__ __forceinline__ void fill_op(const FillPyr& P, int op, int lv, int b, size_t q, int colour) {
  switch (op) {
    case kRestrictInit: restrict_init<C>(P, lv, b, q); break;
    case kProlongInit: prolong_init<C>(P, lv, b, q); break;
    case kDirichlet: dirichlet<C>(P, lv, b, q, colour); break;
    case kCorrect: correct<C>(P, lv, b, q, colour); break;
    case kResidualDown: residual_down<C>(P, lv, b, q); break;
    default: prolong_add<C>(P, lv, b, q); break;
  }
}

// One step over every pixel of level `over` (grid: pixels, fields).
template <int C>
__global__ void __launch_bounds__(kFillThreads) fill_level_kernel(FillPyr P, int op, int lv, int over, int colour) {
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= (size_t)P.l[over].h * P.l[over].w) return;
  fill_op<C>(P, op, lv, blockIdx.y, q, colour);
}

// The rest of a V-cycle from level ls (whose right-hand side and zero correction are written) down to 1 x 1 and back,
// one CTA per field: every step is a pass over one small level, separated by barriers.
template <int C>
__global__ void __launch_bounds__(kFillSmallThreads) fill_small_kernel(FillPyr P, int ls, int smooth) {
  const int b = blockIdx.x;
  auto pass = [&](int op, int lv, int over, int colour) {
    const size_t n = (size_t)P.l[over].h * P.l[over].w;
    for (size_t q = threadIdx.x; q < n; q += blockDim.x) fill_op<C>(P, op, lv, b, q, colour);
    __syncthreads();
  };
  auto sweeps = [&](int lv) {
    for (int s = 0; s < smooth; ++s) {
      pass(kCorrect, lv, lv, 0);
      pass(kCorrect, lv, lv, 1);
    }
  };
  for (int lv = ls; lv < P.L; ++lv) {
    sweeps(lv);
    if (lv + 1 < P.L) pass(kResidualDown, lv, lv + 1, 0);
  }
  for (int lv = P.L - 1; lv >= ls; --lv) {
    if (lv + 1 < P.L) pass(kProlongAdd, lv, lv, 0);
    sweeps(lv);
  }
}

// Per field: the known range of each channel, and the flag of a field without a known pixel (its holes become 0).
// min / max are exact in any order, so the reduction is deterministic.
template <int C>
__global__ void __launch_bounds__(kFillThreads) fill_range_kernel(float* __restrict__ v, const uint8_t* __restrict__ hole,
                                                                  size_t npix, float* __restrict__ lohi,
                                                                  uint8_t* __restrict__ flags) {
  __shared__ float slo[C][kFillThreads], shi[C][kFillThreads];
  __shared__ int sn[kFillThreads];
  const int b = blockIdx.x, t = threadIdx.x;
  float* fv = v + (size_t)b * npix * C;
  const uint8_t* fh = hole + (size_t)b * npix;
  float lo[C], hi[C];
  int n = 0;
  for (size_t q = t; q < npix; q += kFillThreads) {
    if (fh[q]) continue;
#pragma unroll
    for (int c = 0; c < C; ++c) {
      const float x = fv[q * C + c];
      lo[c] = n == 0 ? x : fminf(lo[c], x);
      hi[c] = n == 0 ? x : fmaxf(hi[c], x);
    }
    ++n;
  }
#pragma unroll
  for (int c = 0; c < C; ++c) {
    slo[c][t] = n ? lo[c] : INFINITY;
    shi[c][t] = n ? hi[c] : -INFINITY;
  }
  sn[t] = n;
  __syncthreads();
  for (int h = kFillThreads / 2; h > 0; h >>= 1) {
    if (t < h) {
#pragma unroll
      for (int c = 0; c < C; ++c) {
        slo[c][t] = fminf(slo[c][t], slo[c][t + h]);
        shi[c][t] = fmaxf(shi[c][t], shi[c][t + h]);
      }
      sn[t] = sn[t] || sn[t + h];
    }
    __syncthreads();
  }
  const bool any = sn[0] != 0;
  if (t == 0) {
#pragma unroll
    for (int c = 0; c < C; ++c) {
      lohi[(size_t)b * 2 * C + c] = any ? slo[c][0] : 0.f;
      lohi[(size_t)b * 2 * C + C + c] = any ? shi[c][0] : 0.f;
    }
    if (flags) flags[b] = any ? 0 : 1;
  }
  if (!any) {
    for (size_t q = t; q < npix * C; q += kFillThreads) fv[q] = 0.f;
  }
}

// ---- F25: masks and the temporal fill ----

// A frame pixel is a hole when some pixel of the (2 dilate + 1)^2 square around it has a selected value.
__global__ void __launch_bounds__(256) inpaint_dilate_kernel(const uint8_t* __restrict__ masks,
                                                             const uint8_t* __restrict__ select, int Hs, int Ws,
                                                             int dilate, uint8_t* __restrict__ hole) {
  const size_t npix = (size_t)Hs * Ws;
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= npix) return;
  const size_t base = (size_t)blockIdx.y * npix;
  const int y = (int)(q / Ws), x = (int)(q % Ws);
  uint8_t h = 0;
  for (int yy = max(y - dilate, 0); yy <= min(y + dilate, Hs - 1) && !h; ++yy)
    for (int xx = max(x - dilate, 0); xx <= min(x + dilate, Ws - 1); ++xx)
      if (__ldg(select + masks[base + (size_t)yy * Ws + xx])) {
        h = 1;
        break;
      }
  hole[base + q] = h;
}

// The network index of frame index y under the pixel-centre rule: floor((y + 0.5) Hn / Hs).
__device__ __forceinline__ int net_index(int y, int Hs, int Hn) {
  return (int)(((2 * (int64_t)y + 1) * Hn) / (2 * (int64_t)Hs));
}

// The frame indices [lo, hi) that map to network index i; the one holding i's centre when none does.
__device__ __forceinline__ void frame_span(int i, int Hs, int Hn, int* lo, int* hi) {
  int y = max((int)(((int64_t)i * Hs) / Hn) - 1, 0);
  while (y < Hs && net_index(y, Hs, Hn) < i) ++y;
  *lo = y;
  while (y < Hs && net_index(y, Hs, Hn) == i) ++y;
  *hi = y;
  if (*lo == *hi) {
    *lo = (int)(((2 * (int64_t)i + 1) * Hs) / (2 * (int64_t)Hn));
    *hi = *lo + 1;
  }
}

__global__ void __launch_bounds__(256) inpaint_grid_kernel(const uint8_t* __restrict__ hole, int Hs, int Ws, int Hn,
                                                           int Wn, uint8_t* __restrict__ hole_net) {
  const size_t nn = (size_t)Hn * Wn;
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= nn) return;
  const int i = (int)(q / Wn), j = (int)(q % Wn);
  const uint8_t* h = hole + (size_t)blockIdx.y * Hs * Ws;
  int y0, y1, x0, x1;
  frame_span(i, Hs, Hn, &y0, &y1);
  frame_span(j, Ws, Wn, &x0, &x1);
  uint8_t out = 0;
  for (int y = y0; y < y1 && !out; ++y)
    for (int x = x0; x < x1; ++x)
      if (h[(size_t)y * Ws + x]) {
        out = 1;
        break;
      }
  hole_net[(size_t)blockIdx.y * nn + q] = out;
}

// One side of hole pixel p (network position p0) of frame t: up to n chain steps (dir = +1 forward, -1 backward), each
// followed by the visibility test of the position's four taps in the frame reached.  Returns the distance (0: not
// found) and the colour.
__device__ __forceinline__ int inpaint_side(const uint8_t* __restrict__ frames, const uint8_t* __restrict__ hole,
                                            const float2* __restrict__ fw, const float2* __restrict__ bw, int t, int dir,
                                            int n, float2 p, int Hs, int Ws, int Hn, int Wn, const NetGeom& g,
                                            float s, float a1, float a2, float* col) {
  const size_t nn = (size_t)Hn * Wn, ns = (size_t)Hs * Ws;
  for (int step = 1; step <= n; ++step) {
    const ChainLink l = chain_link(fw, bw, nn, t, dir, step);
    float2 q;
    if (chain_step(l.pull, l.test, Hn, Wn, s, a1, a2, p, q)) return 0;
    p = q;
    const int fr = t + dir * step;
    const Bilerp b = bilerp_at(px_remap(p.x, g.rxs, Ws), px_remap(p.y, g.rys, Hs), Hs, Ws);
    const uint8_t* h = hole + (size_t)fr * ns;
    if (h[(size_t)b.y0 * Ws + b.x0] | h[(size_t)b.y0 * Ws + b.x1] | h[(size_t)b.y1 * Ws + b.x0] |
        h[(size_t)b.y1 * Ws + b.x1])
      continue;
    sample_rgb(frames + (size_t)fr * ns * 3, Ws, b, col);
    return step;
  }
  return 0;
}

// One thread per frame pixel, blockIdx.y over the rows (striding); row r = (t, nf, nb).
__global__ void __launch_bounds__(256) inpaint_propagate_kernel(
    const uint8_t* __restrict__ frames, const uint8_t* __restrict__ hole, int F, int Hs, int Ws,
    const float2* __restrict__ fw, const float2* __restrict__ bw, int Hn, int Wn, NetGeom g, float s, float a1,
    float a2, const int32_t* __restrict__ rows, int n_rows, float* __restrict__ colour, uint8_t* __restrict__ status) {
  const size_t ns = (size_t)Hs * Ws;
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= ns) return;
  const int x = (int)(q % Ws), y = (int)(q / Ws);
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
    const uint8_t* img = frames + ((size_t)t * ns + q) * 3;
    if (!hole[(size_t)t * ns + q]) {
#pragma unroll
      for (int c = 0; c < 3; ++c) out[c] = (float)img[c];
      *st = 0;
      continue;
    }
    const float2 p = make_float2(px_remap(x, g.rxn, Wn), px_remap(y, g.ryn, Hn));
    float cf[3], cb[3];
    const int df = inpaint_side(frames, hole, fw, bw, t, 1, min(max(nf, 0), F - 1 - t), p, Hs, Ws, Hn, Wn, g, s, a1,
                                a2, cf);
    const int db = inpaint_side(frames, hole, fw, bw, t, -1, min(max(nb, 0), t), p, Hs, Ws, Hn, Wn, g, s, a1, a2, cb);
    blend_sides(df, cf, db, cb, out, st);
  }
}

}  // namespace rb

using namespace rb;

namespace {

int fill_levels(int H, int W, int* h, int* w) {
  int L = 0;
  h[0] = H;
  w[0] = W;
  while (!(h[L] == 1 && w[L] == 1)) {
    h[L + 1] = (h[L] + 1) / 2;
    w[L + 1] = (w[L] + 1) / 2;
    ++L;
  }
  return L + 1;
}

size_t align256(size_t x) { return (x + 255) & ~size_t(255); }

// The workspace: per level 1 .. L-1 values, right-hand side and mask of all B fields, then the ranges.
size_t fill_workspace(int B, int C, int L, const int* h, const int* w, size_t* off) {
  size_t at = 0;
  for (int l = 1; l < L; ++l) {
    const size_t n = (size_t)B * h[l] * w[l];
    off[3 * l] = at;
    at += align256(n * C * sizeof(float));
    off[3 * l + 1] = at;
    at += align256(n * C * sizeof(float));
    off[3 * l + 2] = at;
    at += align256(n);
  }
  off[0] = at;
  return at + align256((size_t)B * 2 * C * sizeof(float));
}

template <int C>
int fill_run(float* values, const uint8_t* hole, int B, int H, int W, uint8_t* flags, char* ws, int L, const int* h,
             const int* w, const size_t* off, cudaStream_t st) {
  FillPyr P;
  P.L = L;
  P.l[0] = FillLevel{values, nullptr, const_cast<uint8_t*>(hole), H, W};
  for (int l = 1; l < L; ++l)
    P.l[l] = FillLevel{reinterpret_cast<float*>(ws + off[3 * l]), reinterpret_cast<float*>(ws + off[3 * l + 1]),
                       reinterpret_cast<uint8_t*>(ws + off[3 * l + 2]), h[l], w[l]};
  float* lohi = reinterpret_cast<float*>(ws + off[0]);
  P.lohi = lohi;
  fill_range_kernel<C><<<B, kFillThreads, 0, st>>>(values, hole, (size_t)H * W, lohi, flags);
  RB_CHECK_LAUNCH("fill_range_kernel");
  auto level = [&](int op, int lv, int over, int colour) -> int {
    const size_t n = (size_t)h[over] * w[over];
    fill_level_kernel<C><<<dim3((unsigned)((n + kFillThreads - 1) / kFillThreads), (unsigned)B), kFillThreads, 0, st>>>(
        P, op, lv, over, colour);
    RB_CHECK_LAUNCH("fill_level_kernel");
    return RB_OK;
  };
#define RB_FILL_STEP(...)                \
  do {                                   \
    const int rc_ = level(__VA_ARGS__);  \
    if (rc_ != RB_OK) return rc_;        \
  } while (0)
  for (int l = 1; l < L; ++l) RB_FILL_STEP(kRestrictInit, l, l, 0);
  for (int l = L - 2; l >= 0; --l) {
    RB_FILL_STEP(kProlongInit, l, l, 0);
    for (int s = 0; s < RB_FILL_INIT_SWEEPS; ++s) {
      RB_FILL_STEP(kDirichlet, l, l, 0);
      RB_FILL_STEP(kDirichlet, l, l, 1);
    }
  }
  if (L < 2) return RB_OK;
  int ls = 1;
  while ((size_t)h[ls] * w[ls] > (size_t)kFillSmall) ++ls;
  for (int cyc = 0; cyc < RB_FILL_CYCLES; ++cyc) {
    for (int l = 0; l < ls; ++l) {
      for (int s = 0; l > 0 && s < RB_FILL_SMOOTH; ++s) {
        RB_FILL_STEP(kCorrect, l, l, 0);
        RB_FILL_STEP(kCorrect, l, l, 1);
      }
      RB_FILL_STEP(kResidualDown, l, l + 1, 0);
    }
    fill_small_kernel<C><<<B, kFillSmallThreads, 0, st>>>(P, ls, RB_FILL_SMOOTH);
    RB_CHECK_LAUNCH("fill_small_kernel");
    for (int l = ls - 1; l >= 0; --l) {
      RB_FILL_STEP(kProlongAdd, l, l, 0);
      for (int s = 0; s < RB_FILL_SMOOTH; ++s) {
        RB_FILL_STEP(l > 0 ? kCorrect : kDirichlet, l, l, 0);
        RB_FILL_STEP(l > 0 ? kCorrect : kDirichlet, l, l, 1);
      }
    }
  }
#undef RB_FILL_STEP
  return RB_OK;
}

}  // namespace

extern "C" int rb_masked_fill_workspace_bytes(int B, int H, int W, int C, size_t* bytes) {
  RB_REQUIRE(bytes, RB_ERR_BAD_ARG, "rb_masked_fill_workspace_bytes: null pointer");
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_masked_fill_workspace_bytes: bad shape B=%d H=%d W=%d", B,
             H, W);
  RB_REQUIRE(C == 2 || C == 3, RB_ERR_BAD_ARG, "rb_masked_fill_workspace_bytes: C must be 2 or 3 (got %d)", C);
  int h[kFillMaxLevels], w[kFillMaxLevels];
  size_t off[3 * kFillMaxLevels];
  const int L = fill_levels(H, W, h, w);
  *bytes = fill_workspace(B, C, L, h, w, off);
  return RB_OK;
}

extern "C" int rb_masked_fill(float* values, const uint8_t* hole, int B, int H, int W, int C, uint8_t* flags,
                              void* workspace, size_t workspace_bytes, void* stream) {
  RB_REQUIRE(values && hole && workspace, RB_ERR_BAD_ARG, "rb_masked_fill: null pointer");
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_masked_fill: bad shape B=%d H=%d W=%d", B, H, W);
  RB_REQUIRE(C == 2 || C == 3, RB_ERR_BAD_ARG, "rb_masked_fill: C must be 2 or 3 (got %d)", C);
  RB_REQUIRE(B <= 65535 && (size_t)H * W < (size_t(1) << 31), RB_ERR_BAD_SHAPE,
             "rb_masked_fill: B=%d fields of %dx%d pixels exceed one grid", B, H, W);
  int h[kFillMaxLevels], w[kFillMaxLevels];
  size_t off[3 * kFillMaxLevels];
  const int L = fill_levels(H, W, h, w);
  const size_t need = fill_workspace(B, C, L, h, w, off);
  RB_REQUIRE(workspace_bytes >= need, RB_ERR_WORKSPACE, "rb_masked_fill: workspace of %zu bytes, %zu needed",
             workspace_bytes, need);
  char* ws = static_cast<char*>(workspace);
  const cudaStream_t st = (cudaStream_t)stream;
  return C == 2 ? fill_run<2>(values, hole, B, H, W, flags, ws, L, h, w, off, st)
                : fill_run<3>(values, hole, B, H, W, flags, ws, L, h, w, off, st);
}

extern "C" int rb_inpaint_masks(const uint8_t* masks, const uint8_t* select, int F, int Hs, int Ws, int dilate, int Hn,
                                int Wn, uint8_t* hole, uint8_t* hole_net, void* stream) {
  RB_REQUIRE(masks && select && hole && hole_net, RB_ERR_BAD_ARG, "rb_inpaint_masks: null pointer");
  RB_REQUIRE(F > 0 && Hs > 0 && Ws > 0 && Hn > 0 && Wn > 0, RB_ERR_BAD_SHAPE,
             "rb_inpaint_masks: bad shape F=%d Hs=%d Ws=%d Hn=%d Wn=%d", F, Hs, Ws, Hn, Wn);
  RB_REQUIRE(F <= 65535 && (size_t)Hs * Ws < (size_t(1) << 31) && (size_t)Hn * Wn < (size_t(1) << 31),
             RB_ERR_BAD_SHAPE, "rb_inpaint_masks: F=%d frames of %dx%d exceed one grid", F, Hs, Ws);
  RB_REQUIRE(dilate >= 0 && dilate <= RB_INPAINT_MAX_DILATE, RB_ERR_BAD_ARG,
             "rb_inpaint_masks: dilate must be in [0, %d] (got %d)", RB_INPAINT_MAX_DILATE, dilate);
  RB_REQUIRE(masks != hole, RB_ERR_BAD_ARG, "rb_inpaint_masks: hole must not alias masks");
  const cudaStream_t st = (cudaStream_t)stream;
  const size_t ns = (size_t)Hs * Ws, nn = (size_t)Hn * Wn;
  inpaint_dilate_kernel<<<dim3((unsigned)((ns + 255) / 256), (unsigned)F), 256, 0, st>>>(masks, select, Hs, Ws, dilate,
                                                                                       hole);
  RB_CHECK_LAUNCH("inpaint_dilate_kernel");
  inpaint_grid_kernel<<<dim3((unsigned)((nn + 255) / 256), (unsigned)F), 256, 0, st>>>(hole, Hs, Ws, Hn, Wn, hole_net);
  RB_CHECK_LAUNCH("inpaint_grid_kernel");
  return RB_OK;
}

extern "C" int rb_inpaint_propagate(const uint8_t* frames, const uint8_t* hole, int F, int Hs, int Ws,
                                    const float* flow_fw, const float* flow_bw, int Hn, int Wn, float flow_scale,
                                    float alpha1, float alpha2, const int32_t* rows, int n_rows, float* colour,
                                    uint8_t* status, void* stream) {
  const char* fn = "rb_inpaint_propagate";
  if (int rc = check_rows_entry(fn, frames && hole && rows && colour && status, flow_fw, flow_bw, F, Hs, Ws, Hn, Wn,
                                n_rows))
    return rc;
  if (int rc = check_rows_step(fn, Hs, Ws, flow_scale, alpha1, alpha2)) return rc;
  inpaint_propagate_kernel<<<rows_grid(Hs, Ws, 256, n_rows), 256, 0, (cudaStream_t)stream>>>(
      frames, hole, F, Hs, Ws, reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw), Hn,
      Wn, net_geom(Hs, Ws, Hn, Wn), flow_scale, alpha1, alpha2, rows, n_rows, colour, status);
  RB_CHECK_LAUNCH("inpaint_propagate_kernel");
  return RB_OK;
}
