// F29 - F31: blind video temporal consistency (Bonneel et al., SIGGRAPH Asia 2015) and the warping error of Lai et al.
// (ECCV 2018).  rb_tcons_terms forms each pixel's temporal term from one backward step of the tracker, rb_screened_poisson
// solves the screened Poisson system of the correction with flexible conjugate gradients preconditioned by a multigrid
// V-cycle, and rb_warp_error sums the per-pair warping error.  Every fp32 operation is rounded on its own (__fadd_rn /
// __fmul_rn / __fsub_rn / __fdiv_rn, no FMA contraction) and every reduction runs in a fixed tree, so a numpy
// restatement reproduces the bits (tests/tcons_oracle.py).  No atomics, no allocation.
#include <math.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "fb_sample.cuh"

namespace rb {

constexpr int kTconsThreads = 256;
constexpr int kDotPerThread = 4;
constexpr int kDotChunk = kTconsThreads * kDotPerThread;  // pixels per block of a dot product
constexpr int kWarpPerThread = 16;
constexpr int kWarpChunk = kTconsThreads * kWarpPerThread;  // pixels per block of the warping error

// Fixed-shape tree over the block: s[t] += s[t + h] for h = 128, 64, ..., 1.
__device__ __forceinline__ double tc_block_sum(double v, double* s) {
  const int t = threadIdx.x;
  s[t] = v;
  __syncthreads();
#pragma unroll
  for (int h = kTconsThreads / 2; h > 0; h >>= 1) {
    if (t < h) s[t] = __dadd_rn(s[t], s[t + h]);
    __syncthreads();
  }
  const double r = s[0];
  __syncthreads();
  return r;
}

// One chain step of pixel (x, y) of a frame through pull (tested against test) on the network grid, mapped back to the
// frame: true and the bilinear taps of the target when the step stays on the grid and passes the F5 test.
__device__ __forceinline__ bool tc_step(const float2* __restrict__ pull, const float2* __restrict__ test, int x, int y,
                                        int Hs, int Ws, int Hn, int Wn, const NetGeom& g, float s, float a1, float a2,
                                        Bilerp& b) {
  const float2 p = make_float2(px_remap(x, g.rxn, Wn), px_remap(y, g.ryn, Hn));
  float2 q;
  if (chain_step(pull, test, Hn, Wn, s, a1, a2, p, q)) return false;
  b = bilerp_at(px_remap(q.x, g.rxs, Ws), px_remap(q.y, g.rys, Hs), Hs, Ws);
  return true;
}

// ---- F29 ----
__global__ void __launch_bounds__(kTconsThreads) tcons_terms_kernel(
    const uint8_t* __restrict__ It, const uint8_t* __restrict__ Ip, const uint8_t* __restrict__ Pt,
    const uint8_t* __restrict__ Op, const float2* __restrict__ fw, const float2* __restrict__ bw, int Hs, int Ws,
    int Hn, int Wn, NetGeom g, float s, float a1, float a2, float lam, float* __restrict__ c,
    float* __restrict__ r, uint8_t* __restrict__ status) {
  const size_t ns = (size_t)Hs * Ws;
  const size_t q = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= ns) return;
  const int x = (int)(q % Ws), y = (int)(q / Ws);
  uint8_t st = 3;
  float w = 0.f, ro[3] = {0.f, 0.f, 0.f};
  Bilerp b;
  if (Ip == nullptr) {
    st = 3;
  } else if (!tc_step(bw, fw, x, y, Hs, Ws, Hn, Wn, g, s, a1, a2, b)) {
    st = 1;
  } else {
    float d = 0.f;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float e = __fsub_rn((float)It[q * 3 + ch], sample_rgb1(Ip, Ws, b, ch));
      d = __fadd_rn(d, __fmul_rn(e, e));
    }
    d = __fdiv_rn(d, 3.f);
    const float kk = __fmul_rn(RB_TCONS_KAPPA, RB_TCONS_KAPPA);
    const float xr = __fdiv_rn(d, kk);
    if (xr < 1.f) {
      const float om = __fsub_rn(1.f, xr);
      w = __fmul_rn(om, om);
      st = 0;
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) ro[ch] = __fsub_rn(sample_rgb1(Op, Ws, b, ch), (float)Pt[q * 3 + ch]);
    } else {
      st = 2;
    }
  }
  const float lw = __fmul_rn(lam, w);
  c[q] = __fadd_rn(lw, RB_TCONS_EPS);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) r[q * 3 + ch] = st == 0 ? __fmul_rn(lw, ro[ch]) : 0.f;
  status[q] = st;
}

// ---- F30: the level operators ----
// s = f + e_up + e_down + e_left + e_right (0 for a neighbour outside the level) and the neighbour count n
__device__ __forceinline__ void tc_nbsum(const float* __restrict__ e, const float* __restrict__ f, int h, int w, int x,
                                         int y, float (&s)[3], float& n) {
  const size_t i = (size_t)y * w + x;
  const bool ok[4] = {y > 0, y < h - 1, x > 0, x < w - 1};
  const size_t nb[4] = {i - w, i + w, i - 1, i + 1};
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) s[ch] = f ? f[i * 3 + ch] : 0.f;
  n = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) s[ch] = __fadd_rn(s[ch], ok[k] ? e[nb[k] * 3 + ch] : 0.f);
    n = __fadd_rn(n, ok[k] ? 1.f : 0.f);
  }
}

// res = s - (n e + c e)
__device__ __forceinline__ void tc_resid(const float* __restrict__ c, const float* __restrict__ f,
                                         const float* __restrict__ e, int h, int w, int x, int y, float (&res)[3]) {
  float s[3], n;
  tc_nbsum(e, f, h, w, x, y, s, n);
  const size_t i = (size_t)y * w + x;
  const float ci = c[i];
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float v = e[i * 3 + ch];
    res[ch] = __fsub_rn(s[ch], __fadd_rn(__fmul_rn(n, v), __fmul_rn(ci, v)));
  }
}

// one colour of a red-black Gauss-Seidel sweep: e_p = s / (c_p + n_p) on the pixels with (x + y) % 2 == colour
__global__ void __launch_bounds__(kTconsThreads) tc_sweep_kernel(const float* __restrict__ c, const float* __restrict__ f,
                                                                  float* __restrict__ e, int h, int w, int colour) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)h * w) return;
  const int x = (int)(i % w), y = (int)(i / w);
  if (((x + y) & 1) != colour) return;
  float s[3], n;
  tc_nbsum(e, f, h, w, x, y, s, n);
  const float diag = __fadd_rn(c[i], n);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) e[i * 3 + ch] = __fdiv_rn(s[ch], diag);
}

// coarse pixel (i, j): 0 + the children (2i,2j), (2i,2j+1), (2i+1,2j), (2i+1,2j+1) inside the finer level, in this order
__global__ void __launch_bounds__(kTconsThreads) tc_restrict_c_kernel(const float* __restrict__ cf, int hf, int wf,
                                                                       float* __restrict__ cc, int hc, int wc) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)hc * wc) return;
  const int x = (int)(i % wc), y = (int)(i / wc);
  float v = 0.f;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int cy = 2 * y + (k >> 1), cx = 2 * x + (k & 1);
    if (cy < hf && cx < wf) v = __fadd_rn(v, cf[(size_t)cy * wf + cx]);
  }
  cc[i] = v;
}

// the coarse right-hand side: 0 + the residuals of the children in tap order; the coarse correction starts at 0
__global__ void __launch_bounds__(kTconsThreads) tc_restrict_kernel(const float* __restrict__ c,
                                                                     const float* __restrict__ f,
                                                                     const float* __restrict__ e, int hf, int wf,
                                                                     float* __restrict__ fc, float* __restrict__ ec,
                                                                     int hc, int wc) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)hc * wc) return;
  const int x = (int)(i % wc), y = (int)(i / wc);
  float v[3] = {0.f, 0.f, 0.f};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int cy = 2 * y + (k >> 1), cx = 2 * x + (k & 1);
    if (cy < hf && cx < wf) {
      float res[3];
      tc_resid(c, f, e, hf, wf, cx, cy, res);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) v[ch] = __fadd_rn(v[ch], res[ch]);
    }
  }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    fc[i * 3 + ch] = v[ch];
    ec[i * 3 + ch] = 0.f;
  }
}

__device__ __forceinline__ void tc_taps(int z, int n, int& a, int& b, float& wa, float& wb) {
  const int i = z >> 1;
  if ((z & 1) == 0) {
    a = max(i - 1, 0);
    b = i;
    wa = 0.25f;
    wb = 0.75f;
  } else {
    a = i;
    b = min(i + 1, n - 1);
    wa = 0.75f;
    wb = 0.25f;
  }
}

// e_f += the cell-centred bilinear value of the coarse correction: ((wxa e_aa + wxb e_ab) wya) + ((wxa e_ba + wxb e_bb) wyb)
__global__ void __launch_bounds__(kTconsThreads) tc_prolong_kernel(const float* __restrict__ ec, int hc, int wc,
                                                                    float* __restrict__ ef, int hf, int wf) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)hf * wf) return;
  const int x = (int)(i % wf), y = (int)(i / wf);
  int xa, xb, ya, yb;
  float wxa, wxb, wya, wyb;
  tc_taps(x, wc, xa, xb, wxa, wxb);
  tc_taps(y, hc, ya, yb, wya, wyb);
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const float t0 = __fadd_rn(__fmul_rn(wxa, ec[((size_t)ya * wc + xa) * 3 + ch]),
                               __fmul_rn(wxb, ec[((size_t)ya * wc + xb) * 3 + ch]));
    const float t1 = __fadd_rn(__fmul_rn(wxa, ec[((size_t)yb * wc + xa) * 3 + ch]),
                               __fmul_rn(wxb, ec[((size_t)yb * wc + xb) * 3 + ch]));
    ef[i * 3 + ch] = __fadd_rn(ef[i * 3 + ch], __fadd_rn(__fmul_rn(t0, wya), __fmul_rn(t1, wyb)));
  }
}

// ---- F30: the Krylov pieces ----
// q = A p (A p = (c + n) p - sum of the neighbours' p, as -(s - (n p + c p)) with f = 0) and the block partials of <p, q>
__global__ void __launch_bounds__(kTconsThreads) tc_matvec_dot_kernel(const float* __restrict__ c,
                                                                       const float* __restrict__ p,
                                                                       float* __restrict__ q, int H, int W,
                                                                       double* __restrict__ partials) {
  __shared__ double red[kTconsThreads];
  const size_t N = (size_t)H * W;
  double acc[3] = {0.0, 0.0, 0.0};
#pragma unroll
  for (int k = 0; k < kDotPerThread; ++k) {
    const size_t i = (size_t)blockIdx.x * kDotChunk + (size_t)k * kTconsThreads + threadIdx.x;
    if (i < N) {
      float res[3];
      tc_resid(c, nullptr, p, H, W, (int)(i % W), (int)(i / W), res);
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) {
        const float v = -res[ch];
        q[i * 3 + ch] = v;
        acc[ch] = __dadd_rn(acc[ch], __dmul_rn((double)p[i * 3 + ch], (double)v));
      }
    } else {
#pragma unroll
      for (int ch = 0; ch < 3; ++ch) acc[ch] = __dadd_rn(acc[ch], 0.0);
    }
  }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const double v = tc_block_sum(acc[ch], red);
    if (threadIdx.x == 0) partials[(size_t)blockIdx.x * 3 + ch] = v;
  }
}

// block partials of <a, b> (and of <a2, b2> into partials2 when a2 is given)
__global__ void __launch_bounds__(kTconsThreads) tc_dot_kernel(const float* __restrict__ a, const float* __restrict__ b,
                                                                const float* __restrict__ a2,
                                                                const float* __restrict__ b2, size_t N,
                                                                double* __restrict__ partials,
                                                                double* __restrict__ partials2) {
  __shared__ double red[kTconsThreads];
  double acc[3] = {0.0, 0.0, 0.0}, acc2[3] = {0.0, 0.0, 0.0};
#pragma unroll
  for (int k = 0; k < kDotPerThread; ++k) {
    const size_t i = (size_t)blockIdx.x * kDotChunk + (size_t)k * kTconsThreads + threadIdx.x;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const bool in = i < N;
      acc[ch] = __dadd_rn(acc[ch], in ? __dmul_rn((double)a[i * 3 + ch], (double)b[i * 3 + ch]) : 0.0);
      if (a2) acc2[ch] = __dadd_rn(acc2[ch], in ? __dmul_rn((double)a2[i * 3 + ch], (double)b2[i * 3 + ch]) : 0.0);
    }
  }
#pragma unroll
  for (int ch = 0; ch < 3; ++ch) {
    const double v = tc_block_sum(acc[ch], red);
    if (threadIdx.x == 0) partials[(size_t)blockIdx.x * 3 + ch] = v;
  }
  if (a2) {
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const double v = tc_block_sum(acc2[ch], red);
      if (threadIdx.x == 0) partials2[(size_t)blockIdx.x * 3 + ch] = v;
    }
  }
}

// one block: per channel, thread t adds partials t, t + 256, ... (0 past the end) in order, then the fixed tree
__global__ void __launch_bounds__(kTconsThreads) tc_reduce_kernel(const double* __restrict__ partials, int nb,
                                                                   double* __restrict__ out) {
  __shared__ double red[kTconsThreads];
  const int rounds = (nb + kTconsThreads - 1) / kTconsThreads;
  for (int ch = 0; ch < 3; ++ch) {
    double v = 0.0;
    for (int k = 0; k < rounds; ++k) {
      const int i = k * kTconsThreads + threadIdx.x;
      v = __dadd_rn(v, i < nb ? partials[(size_t)i * 3 + ch] : 0.0);
    }
    const double s = tc_block_sum(v, red);
    if (threadIdx.x == 0) out[ch] = s;
  }
}

// alpha = fl32(rho / pq) (0 unless pq > 0); x += alpha p; res' = res - alpha q; d = res' - res; res = res'
__global__ void __launch_bounds__(kTconsThreads) tc_update_x_kernel(const double* __restrict__ rho,
                                                                     const double* __restrict__ pq,
                                                                     const float* __restrict__ p,
                                                                     const float* __restrict__ q, float* __restrict__ x,
                                                                     float* __restrict__ res, float* __restrict__ d,
                                                                     size_t n3) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n3) return;
  const int ch = (int)(i % 3);
  const double den = pq[ch];
  const float alpha = den > 0.0 ? __double2float_rn(__ddiv_rn(rho[ch], den)) : 0.f;
  x[i] = __fadd_rn(x[i], __fmul_rn(alpha, p[i]));
  const float r0 = res[i];
  const float r1 = __fsub_rn(r0, __fmul_rn(alpha, q[i]));
  res[i] = r1;
  d[i] = __fsub_rn(r1, r0);
}

// beta = fl32(zd / rho) (0 unless rho > 0); p = z + beta p
__global__ void __launch_bounds__(kTconsThreads) tc_update_p_kernel(const double* __restrict__ zd,
                                                                     const double* __restrict__ rho,
                                                                     const float* __restrict__ z, float* __restrict__ p,
                                                                     size_t n3) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n3) return;
  const int ch = (int)(i % 3);
  const double den = rho[ch];
  const float beta = den > 0.0 ? __double2float_rn(__ddiv_rn(zd[ch], den)) : 0.f;
  p[i] = __fadd_rn(z[i], __fmul_rn(beta, p[i]));
}

// ---- F31 ----
// grid (chunks, pairs); thread t takes pixels chunk_start + k * 256 + t, k = 0..15 in order
__global__ void __launch_bounds__(kTconsThreads) warp_error_chunk_kernel(
    const uint8_t* __restrict__ video, int Hs, int Ws, const float2* __restrict__ fw, const float2* __restrict__ bw,
    int Hn, int Wn, NetGeom g, float s, float a1, float a2, double* __restrict__ partials) {
  __shared__ double red[kTconsThreads];
  const int k = blockIdx.y;
  const size_t ns = (size_t)Hs * Ws, nn = (size_t)Hn * Wn;
  const uint8_t* a = video + (size_t)k * ns * 3;
  const uint8_t* b = a + ns * 3;
  double sum = 0.0, cnt = 0.0;
  for (int j = 0; j < kWarpPerThread; ++j) {
    const size_t q = (size_t)blockIdx.x * kWarpChunk + (size_t)j * kTconsThreads + threadIdx.x;
    if (q >= ns) break;
    Bilerp bl;
    if (!tc_step(fw + (size_t)k * nn, bw + (size_t)k * nn, (int)(q % Ws), (int)(q / Ws), Hs, Ws, Hn, Wn, g, s, a1, a2,
                 bl))
      continue;
    float e = 0.f;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
      const float d = __fsub_rn((float)a[q * 3 + ch], sample_rgb1(b, Ws, bl, ch));
      e = __fadd_rn(e, __fmul_rn(d, d));
    }
    sum = __dadd_rn(sum, (double)e);
    cnt = __dadd_rn(cnt, 1.0);
  }
  double* dst = partials + ((size_t)k * gridDim.x + blockIdx.x) * 2;
  const double s0 = tc_block_sum(sum, red);
  const double s1 = tc_block_sum(cnt, red);
  if (threadIdx.x == 0) {
    dst[0] = s0;
    dst[1] = s1;
  }
}

// one block per pair: thread t adds partials t, t + 256, ... in order, then the fixed tree
__global__ void __launch_bounds__(kTconsThreads) warp_error_pair_kernel(const double* __restrict__ partials, int chunks,
                                                                         double* __restrict__ sums) {
  __shared__ double red[kTconsThreads];
  const double* src = partials + (size_t)blockIdx.x * chunks * 2;
  for (int m = 0; m < 2; ++m) {
    double v = 0.0;
    for (int i = threadIdx.x; i < chunks; i += kTconsThreads) v = __dadd_rn(v, src[(size_t)i * 2 + m]);
    const double r = tc_block_sum(v, red);
    if (threadIdx.x == 0) sums[(size_t)blockIdx.x * 2 + m] = r;
  }
}

// ---- F30's workspace ----
std::vector<int2> tc_levels(int H, int W) {
  std::vector<int2> lv{make_int2(H, W)};
  while (lv.back().x != 1 || lv.back().y != 1) {
    const int2 l = lv.back();
    lv.push_back(make_int2((l.x + 1) / 2, (l.y + 1) / 2));
  }
  return lv;
}

size_t tc_align(size_t b) { return (b + 255) & ~size_t(255); }

struct PoissonWs {
  std::vector<float*> c, f, e;  // per level (level 0: c the input, f the residual, e the preconditioned residual z)
  float *p, *q, *d;
  double *part, *part2, *dots;  // dots: [6][3] = rho (two slots), pq, zd
  int nb;
};

size_t tc_poisson_layout(int H, int W, char* base, PoissonWs* ws) {
  const std::vector<int2> lv = tc_levels(H, W);
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += tc_align(bytes);
    return p;
  };
  const size_t n0 = (size_t)H * W;
  const int nb = (int)((n0 + kDotChunk - 1) / kDotChunk);
  if (ws) {
    ws->c.assign(lv.size(), nullptr);
    ws->f.assign(lv.size(), nullptr);
    ws->e.assign(lv.size(), nullptr);
    ws->nb = nb;
  }
  for (size_t l = 0; l < lv.size(); ++l) {
    const size_t n = (size_t)lv[l].x * lv[l].y;
    float* c = l ? (float*)take(n * sizeof(float)) : nullptr;
    float* f = (float*)take(n * 3 * sizeof(float));
    float* e = (float*)take(n * 3 * sizeof(float));
    if (ws) {
      ws->c[l] = c;
      ws->f[l] = f;
      ws->e[l] = e;
    }
  }
  float* p = (float*)take(n0 * 3 * sizeof(float));
  float* q = (float*)take(n0 * 3 * sizeof(float));
  float* d = (float*)take(n0 * 3 * sizeof(float));
  double* part = (double*)take((size_t)nb * 3 * sizeof(double));
  double* part2 = (double*)take((size_t)nb * 3 * sizeof(double));
  double* dots = (double*)take(6 * 3 * sizeof(double));
  if (ws) {
    ws->p = p;
    ws->q = q;
    ws->d = d;
    ws->part = part;
    ws->part2 = part2;
    ws->dots = dots;
  }
  return off;
}

bool tc_overlap(const void* a, size_t na, const void* b, size_t nb) {
  const uintptr_t x = (uintptr_t)a, y = (uintptr_t)b;
  return x < y + nb && y < x + na;
}

unsigned tc_blocks(size_t n) { return (unsigned)((n + kTconsThreads - 1) / kTconsThreads); }

// z = V(f0) on levels lv with the workspace's pyramids (ws.f[0] the right-hand side, ws.e[0] the result)
int tc_vcycle(const std::vector<int2>& lv, const PoissonWs& ws, cudaStream_t st) {
  const int L = (int)lv.size();
  RB_CHECK_CUDA(cudaMemsetAsync(ws.e[0], 0, (size_t)lv[0].x * lv[0].y * 3 * sizeof(float), st));
  auto smooth = [&](int l) {
    const size_t n = (size_t)lv[l].x * lv[l].y;
    for (int k = 0; k < RB_TCONS_SWEEPS; ++k)
      for (int colour = 0; colour < 2; ++colour)
        tc_sweep_kernel<<<tc_blocks(n), kTconsThreads, 0, st>>>(ws.c[l], ws.f[l], ws.e[l], lv[l].x, lv[l].y, colour);
  };
  for (int l = 0; l + 1 < L; ++l) {
    smooth(l);
    const size_t nc = (size_t)lv[l + 1].x * lv[l + 1].y;
    tc_restrict_kernel<<<tc_blocks(nc), kTconsThreads, 0, st>>>(ws.c[l], ws.f[l], ws.e[l], lv[l].x, lv[l].y,
                                                                ws.f[l + 1], ws.e[l + 1], lv[l + 1].x, lv[l + 1].y);
  }
  smooth(L - 1);
  for (int l = L - 2; l >= 0; --l) {
    tc_prolong_kernel<<<tc_blocks((size_t)lv[l].x * lv[l].y), kTconsThreads, 0, st>>>(
        ws.e[l + 1], lv[l + 1].x, lv[l + 1].y, ws.e[l], lv[l].x, lv[l].y);
    smooth(l);
  }
  RB_CHECK_LAUNCH("tc_vcycle");
  return RB_OK;
}

}  // namespace rb

using namespace rb;

extern "C" int rb_tcons_terms(const uint8_t* frame, const uint8_t* prev_frame, const uint8_t* processed,
                              const uint8_t* prev_out, int Hs, int Ws, const float* flow_fw, const float* flow_bw,
                              int Hn, int Wn, float flow_scale, float alpha1, float alpha2, float strength, float* c,
                              float* r, uint8_t* status, void* stream) {
  RB_REQUIRE(c && r && status, RB_ERR_BAD_ARG, "rb_tcons_terms: null output");
  RB_REQUIRE(!prev_frame || (frame && processed && prev_out && flow_fw && flow_bw), RB_ERR_BAD_ARG,
             "rb_tcons_terms: null pointer");
  RB_REQUIRE(Hs > 0 && Ws > 0 && Hn > 0 && Wn > 0, RB_ERR_BAD_SHAPE, "rb_tcons_terms: bad shape Hs=%d Ws=%d Hn=%d Wn=%d",
             Hs, Ws, Hn, Wn);
  RB_REQUIRE((size_t)Hs * Ws < (size_t(1) << 31), RB_ERR_BAD_SHAPE,
             "rb_tcons_terms: %dx%d pixels per frame exceed one grid", Hs, Ws);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "rb_tcons_terms: flow_scale must be finite and > 0 (got %g)", (double)flow_scale);
  RB_REQUIRE(alpha1 >= 0.f && isfinite(alpha1) && alpha2 >= 0.f && isfinite(alpha2), RB_ERR_BAD_ARG,
             "rb_tcons_terms: alpha1, alpha2 must be finite and >= 0 (got %g, %g)", (double)alpha1, (double)alpha2);
  RB_REQUIRE(strength > 0.f && isfinite(strength), RB_ERR_BAD_ARG,
             "rb_tcons_terms: strength must be finite and > 0 (got %g)", (double)strength);
  const size_t ns = (size_t)Hs * Ws;
  tcons_terms_kernel<<<tc_blocks(ns), kTconsThreads, 0, (cudaStream_t)stream>>>(
      frame, prev_frame, processed, prev_out, reinterpret_cast<const float2*>(flow_fw),
      reinterpret_cast<const float2*>(flow_bw), Hs, Ws, Hn, Wn, net_geom(Hs, Ws, Hn, Wn), flow_scale, alpha1, alpha2,
      strength, c, r, status);
  RB_CHECK_LAUNCH("tcons_terms_kernel");
  return RB_OK;
}

extern "C" int rb_screened_poisson_workspace_bytes(int H, int W, size_t* bytes) {
  RB_REQUIRE(bytes, RB_ERR_BAD_ARG, "rb_screened_poisson_workspace_bytes: null pointer");
  RB_REQUIRE(H > 0 && W > 0 && (size_t)H * W < (size_t(1) << 31), RB_ERR_BAD_SHAPE,
             "rb_screened_poisson_workspace_bytes: bad shape H=%d W=%d", H, W);
  *bytes = tc_poisson_layout(H, W, nullptr, nullptr);
  return RB_OK;
}

extern "C" int rb_screened_poisson(const float* c, const float* r, int H, int W, float* D, void* workspace,
                                   size_t workspace_bytes, void* stream) {
  RB_REQUIRE(c && r && D && workspace, RB_ERR_BAD_ARG, "rb_screened_poisson: null pointer");
  RB_REQUIRE(H > 0 && W > 0 && (size_t)H * W < (size_t(1) << 31), RB_ERR_BAD_SHAPE,
             "rb_screened_poisson: bad shape H=%d W=%d", H, W);
  const size_t need = tc_poisson_layout(H, W, nullptr, nullptr);
  const size_t n3b = (size_t)H * W * 3 * sizeof(float);
  RB_REQUIRE(!tc_overlap(D, n3b, r, n3b) && !tc_overlap(D, n3b, c, n3b / 3) && !tc_overlap(D, n3b, workspace, need) &&
                 !tc_overlap(workspace, need, r, n3b) && !tc_overlap(workspace, need, c, n3b / 3),
             RB_ERR_BAD_ARG, "rb_screened_poisson: D, c, r and the workspace must not overlap");
  RB_REQUIRE(workspace_bytes >= need, RB_ERR_BAD_ARG, "rb_screened_poisson: workspace of %zu bytes, %zu needed",
             workspace_bytes, need);
  const cudaStream_t st = (cudaStream_t)stream;
  const std::vector<int2> lv = tc_levels(H, W);
  PoissonWs ws;
  tc_poisson_layout(H, W, (char*)workspace, &ws);
  ws.c[0] = const_cast<float*>(c);  // read only
  const size_t n0 = (size_t)H * W, n3 = n0 * 3;
  for (size_t l = 1; l < lv.size(); ++l)
    tc_restrict_c_kernel<<<tc_blocks((size_t)lv[l].x * lv[l].y), kTconsThreads, 0, st>>>(
        ws.c[l - 1], lv[l - 1].x, lv[l - 1].y, ws.c[l], lv[l].x, lv[l].y);
  float* res = ws.f[0];
  float* z = ws.e[0];
  double* rho[2] = {ws.dots, ws.dots + 3};
  double* pq = ws.dots + 6;
  double* zd = ws.dots + 9;
  RB_CHECK_CUDA(cudaMemsetAsync(D, 0, n3 * sizeof(float), st));
  RB_CHECK_CUDA(cudaMemcpyAsync(res, r, n3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  int rc = tc_vcycle(lv, ws, st);
  if (rc != RB_OK) return rc;
  RB_CHECK_CUDA(cudaMemcpyAsync(ws.p, z, n3 * sizeof(float), cudaMemcpyDeviceToDevice, st));
  tc_dot_kernel<<<ws.nb, kTconsThreads, 0, st>>>(res, z, nullptr, nullptr, n0, ws.part, nullptr);
  tc_reduce_kernel<<<1, kTconsThreads, 0, st>>>(ws.part, ws.nb, rho[0]);
  for (int it = 0; it < RB_TCONS_ITERS; ++it) {
    tc_matvec_dot_kernel<<<ws.nb, kTconsThreads, 0, st>>>(c, ws.p, ws.q, H, W, ws.part);
    tc_reduce_kernel<<<1, kTconsThreads, 0, st>>>(ws.part, ws.nb, pq);
    tc_update_x_kernel<<<tc_blocks(n3), kTconsThreads, 0, st>>>(rho[it & 1], pq, ws.p, ws.q, D, res, ws.d, n3);
    if (it == RB_TCONS_ITERS - 1) break;
    rc = tc_vcycle(lv, ws, st);
    if (rc != RB_OK) return rc;
    tc_dot_kernel<<<ws.nb, kTconsThreads, 0, st>>>(z, ws.d, res, z, n0, ws.part, ws.part2);
    tc_reduce_kernel<<<1, kTconsThreads, 0, st>>>(ws.part, ws.nb, zd);
    tc_reduce_kernel<<<1, kTconsThreads, 0, st>>>(ws.part2, ws.nb, rho[(it + 1) & 1]);
    tc_update_p_kernel<<<tc_blocks(n3), kTconsThreads, 0, st>>>(zd, rho[it & 1], z, ws.p, n3);
  }
  RB_CHECK_LAUNCH("rb_screened_poisson");
  return RB_OK;
}

extern "C" int rb_warp_error_workspace_bytes(int F, int Hs, int Ws, size_t* bytes) {
  RB_REQUIRE(bytes, RB_ERR_BAD_ARG, "rb_warp_error_workspace_bytes: null pointer");
  RB_REQUIRE(F >= 2 && Hs > 0 && Ws > 0 && (size_t)Hs * Ws < (size_t(1) << 31), RB_ERR_BAD_SHAPE,
             "rb_warp_error_workspace_bytes: bad shape F=%d Hs=%d Ws=%d", F, Hs, Ws);
  const size_t chunks = ((size_t)Hs * Ws + kWarpChunk - 1) / kWarpChunk;
  *bytes = (size_t)(F - 1) * chunks * 2 * sizeof(double);
  return RB_OK;
}

extern "C" int rb_warp_error(const uint8_t* video, int F, int Hs, int Ws, const float* flow_fw, const float* flow_bw,
                             int Hn, int Wn, float flow_scale, float alpha1, float alpha2, double* sums,
                             void* workspace, size_t workspace_bytes, void* stream) {
  RB_REQUIRE(video && flow_fw && flow_bw && sums && workspace, RB_ERR_BAD_ARG, "rb_warp_error: null pointer");
  RB_REQUIRE(F >= 2 && Hs > 0 && Ws > 0 && Hn > 0 && Wn > 0, RB_ERR_BAD_SHAPE,
             "rb_warp_error: bad shape F=%d Hs=%d Ws=%d Hn=%d Wn=%d", F, Hs, Ws, Hn, Wn);
  RB_REQUIRE(F - 1 <= 65535 && (size_t)Hs * Ws < (size_t(1) << 31), RB_ERR_BAD_SHAPE,
             "rb_warp_error: %d pairs of %dx%d pixels exceed one grid", F - 1, Hs, Ws);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "rb_warp_error: flow_scale must be finite and > 0 (got %g)", (double)flow_scale);
  RB_REQUIRE(alpha1 >= 0.f && isfinite(alpha1) && alpha2 >= 0.f && isfinite(alpha2), RB_ERR_BAD_ARG,
             "rb_warp_error: alpha1, alpha2 must be finite and >= 0 (got %g, %g)", (double)alpha1, (double)alpha2);
  const size_t chunks = ((size_t)Hs * Ws + kWarpChunk - 1) / kWarpChunk;
  RB_REQUIRE(workspace_bytes >= (size_t)(F - 1) * chunks * 2 * sizeof(double), RB_ERR_BAD_ARG,
             "rb_warp_error: workspace too small (%zu bytes)", workspace_bytes);
  const cudaStream_t st = (cudaStream_t)stream;
  double* part = (double*)workspace;
  warp_error_chunk_kernel<<<dim3((unsigned)chunks, (unsigned)(F - 1)), kTconsThreads, 0, st>>>(
      video, Hs, Ws, reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw), Hn, Wn,
      net_geom(Hs, Ws, Hn, Wn), flow_scale, alpha1, alpha2, part);
  warp_error_pair_kernel<<<F - 1, kTconsThreads, 0, st>>>(part, (int)chunks, sums);
  RB_CHECK_LAUNCH("warp_error_kernels");
  return RB_OK;
}
