// F9: end-point error metrics of a batch of flows against ground truth (upstream RAFT's evaluate.py: validate_sintel /
// validate_kitti).  Two launches, no float atomics: every block reduces one fixed chunk of one sample's pixels in a fixed
// tree and writes its partial sums to the workspace, then one block per sample adds that sample's partials in a fixed
// order.  The chunks are per sample, so a sample's stats do not depend on B or on where it sits in the batch.
#include <math.h>

#include "common.cuh"

namespace rb {

constexpr int kMetricsThreads = 256;
constexpr int kMetricsPerThread = 16;
constexpr int kMetricsChunk = kMetricsThreads * kMetricsPerThread;  // pixels per block
constexpr int kStats = RB_FLOW_STATS;
// fl32(e / m) > 0.05f without the division (whose IEEE slow path is a call that makes ptxas spill): 0.05f = 13421773 * 2^-28
// with an odd significand, so the quotient rounds above it exactly when e / m >= mid = 26843547 * 2^-29, the midpoint to
// the next float (a tie rounds to the even neighbour above).  mid * m has at most 25 + 24 significant bits, so the double
// product is exact and (double)e >= mid * m decides the same as the rounded quotient -- for m = 0 (e > 3 gives +inf),
// m = inf (0), subnormal m and NaN (false) too.
constexpr double kF1Mid = 26843547.0 / 536870912.0;

// Fixed-shape tree over the block: s[t] += s[t + h] for h = 128, 64, ..., 1.
__device__ __forceinline__ double block_sum(double v, double* s) {
  const int t = threadIdx.x;
  s[t] = v;
  __syncthreads();
#pragma unroll
  for (int h = kMetricsThreads / 2; h > 0; h >>= 1) {
    if (t < h) s[t] += s[t + h];
    __syncthreads();
  }
  const double r = s[0];
  __syncthreads();  // s is reused by the next call
  return r;
}

// grid (chunks per sample, B); thread t takes pixels chunk_start + k * 256 + t, k = 0..15 in order (coalesced).
__global__ void __launch_bounds__(kMetricsThreads) flow_metrics_chunk_kernel(
    const float2* __restrict__ flow, float s, const float2* __restrict__ gt, const uint8_t* __restrict__ valid,
    float* __restrict__ epe, double* __restrict__ partials, size_t npix) {
  __shared__ double red[kMetricsThreads];
  const int b = blockIdx.y;
  const size_t base = (size_t)b * npix;
  const size_t c0 = (size_t)blockIdx.x * kMetricsChunk;
  double sum_e = 0.0;
  unsigned n = 0, c1 = 0, c3 = 0, c5 = 0, out = 0;
#pragma unroll 4
  for (int k = 0; k < kMetricsPerThread; ++k) {
    const size_t q = c0 + (size_t)k * kMetricsThreads + threadIdx.x;
    if (q >= npix) break;
    const size_t p = base + q;
    const float2 f = flow[p], g = gt[p];
    // each operation rounded on its own (no FMA contraction): upstream's torch expressions bit for bit
    const float dx = __fsub_rn(__fmul_rn(s, f.x), g.x), dy = __fsub_rn(__fmul_rn(s, f.y), g.y);
    const float e = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
    if (epe) epe[p] = e;
    if (valid && !valid[p]) continue;
    const float m = __fsqrt_rn(__fadd_rn(__fmul_rn(g.x, g.x), __fmul_rn(g.y, g.y)));
    ++n;
    sum_e += (double)e;  // a NaN flow propagates into the sum, as it does upstream
    c1 += e < 1.0f;
    c3 += e < 3.0f;
    c5 += e < 5.0f;
    out += e > 3.0f && (double)e >= __dmul_rn(kF1Mid, (double)m);  // KITTI's F1 outlier: e / m > 0.05f (kF1Mid)
  }
  const double v[kStats] = {(double)n, sum_e, (double)c1, (double)c3, (double)c5, (double)out};
  double* dst = partials + ((size_t)b * gridDim.x + blockIdx.x) * kStats;
#pragma unroll
  for (int i = 0; i < kStats; ++i) {
    const double r = block_sum(v[i], red);
    if (threadIdx.x == 0) dst[i] = r;
  }
}

// one block per sample: thread t adds partials t, t + 256, ... in order, then the fixed tree
__global__ void __launch_bounds__(kMetricsThreads) flow_metrics_sample_kernel(const double* __restrict__ partials,
                                                                              int chunks, double* __restrict__ stats) {
  __shared__ double red[kMetricsThreads];
  const int b = blockIdx.x;
  const double* src = partials + (size_t)b * chunks * kStats;
  double v[kStats] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int c = threadIdx.x; c < chunks; c += kMetricsThreads) {
#pragma unroll
    for (int i = 0; i < kStats; ++i) v[i] += src[(size_t)c * kStats + i];
  }
#pragma unroll
  for (int i = 0; i < kStats; ++i) {
    const double r = block_sum(v[i], red);
    if (threadIdx.x == 0) stats[(size_t)b * kStats + i] = r;
  }
}

static int metrics_chunks(int H, int W) { return (int)(((size_t)H * W + kMetricsChunk - 1) / kMetricsChunk); }

// ---- F12: frame metrics (SSE and SSIM of interpolated frames against ground truth) ------------------------------------
// One block per (kFmTileH x kFmTileW output tile, sample).  The tile plus a kFmR-pixel halo of both images is staged in
// shared memory as uint8 (pred quantised on load; pixels outside the image read as 0 -- they only reach outputs outside
// the SSIM crop, which are not counted).  Per channel: a horizontal pass writes the five weighted row sums of x, y, x^2,
// y^2, xy for every staged row, a vertical pass finishes the 11x11 means and S per output pixel, all in fp64.  The SSE
// is summed exactly (integers) over the tile's pixels, halo excluded.  Partials {sse, sum S} per tile go to the
// workspace in tile order; a second launch adds them per sample in a fixed order, as for the flow metrics.
constexpr int kFmR = 5;                        // window radius: int(3.5 * 1.5 + 0.5), scipy's truncate = 3.5
constexpr int kFmTileW = 32, kFmTileH = 16;    // output tile; 256 threads = 8 rows of 32
constexpr int kFmSW = kFmTileW + 2 * kFmR;     // staged columns
constexpr int kFmSH = kFmTileH + 2 * kFmR;     // staged rows
constexpr int kFmStats = RB_FRAME_STATS;

struct Gauss11 {
  double w[kFmR + 1];  // w[k] = weight of offsets +-k
};

__global__ void __launch_bounds__(kMetricsThreads) frame_metrics_tile_kernel(
    const void* __restrict__ pred, int pred_is_u8, const uint8_t* __restrict__ gt, int H, int W, int tiles_x,
    Gauss11 g, double* __restrict__ partials) {
  __shared__ uint8_t sx[3][kFmSH][kFmSW], sy[3][kFmSH][kFmSW];
  __shared__ double hs[5][kFmSH][kFmTileW];
  __shared__ double red[kMetricsThreads];
  const int b = blockIdx.y, t = threadIdx.x;
  const int x0 = (int)(blockIdx.x % tiles_x) * kFmTileW, y0 = (int)(blockIdx.x / tiles_x) * kFmTileH;
  const size_t base = (size_t)b * H * W * 3;
  unsigned long long sse = 0;
  for (int e = t; e < kFmSH * kFmSW * 3; e += kMetricsThreads) {
    const int c = e % 3, p = e / 3, r = p / kFmSW, col = p % kFmSW;
    const int y = y0 - kFmR + r, x = x0 - kFmR + col;
    uint8_t q = 0, v = 0;
    if (y >= 0 && y < H && x >= 0 && x < W) {
      const size_t i = base + ((size_t)y * W + x) * 3 + c;
      q = pred_is_u8 ? static_cast<const uint8_t*>(pred)[i] : quantise(static_cast<const float*>(pred)[i]);
      v = gt[i];
      if (r >= kFmR && r < kFmR + kFmTileH && col >= kFmR && col < kFmR + kFmTileW) {
        const int d = (int)q - (int)v;
        sse += (unsigned long long)(d * d);
      }
    }
    sx[c][r][col] = q;
    sy[c][r][col] = v;
  }
  __syncthreads();
  double ssim = 0.0;
  constexpr double C1 = (0.01 * 255) * (0.01 * 255), C2 = (0.03 * 255) * (0.03 * 255);
  for (int c = 0; c < 3; ++c) {
    for (int e = t; e < kFmSH * kFmTileW; e += kMetricsThreads) {
      const int r = e / kFmTileW, j = e % kFmTileW;
      const uint8_t* rx = &sx[c][r][j + kFmR];
      const uint8_t* ry = &sy[c][r][j + kFmR];
      double a = (double)rx[0], bb = (double)ry[0];
      double m[5] = {g.w[0] * a, g.w[0] * bb, g.w[0] * (a * a), g.w[0] * (bb * bb), g.w[0] * (a * bb)};
#pragma unroll
      for (int k = 1; k <= kFmR; ++k) {
        const double a0 = rx[-k], a1 = rx[k], b0 = ry[-k], b1 = ry[k];
        m[0] += g.w[k] * (a0 + a1);
        m[1] += g.w[k] * (b0 + b1);
        m[2] += g.w[k] * (a0 * a0 + a1 * a1);
        m[3] += g.w[k] * (b0 * b0 + b1 * b1);
        m[4] += g.w[k] * (a0 * b0 + a1 * b1);
      }
#pragma unroll
      for (int i = 0; i < 5; ++i) hs[i][r][j] = m[i];
    }
    __syncthreads();
    for (int e = t; e < kFmTileH * kFmTileW; e += kMetricsThreads) {
      const int i = e / kFmTileW, j = e % kFmTileW, y = y0 + i, x = x0 + j;
      double m[5];
#pragma unroll
      for (int n = 0; n < 5; ++n) {
        double s = g.w[0] * hs[n][i + kFmR][j];
#pragma unroll
        for (int k = 1; k <= kFmR; ++k) s += g.w[k] * (hs[n][i + kFmR - k][j] + hs[n][i + kFmR + k][j]);
        m[n] = s;
      }
      const double vx = m[2] - m[0] * m[0], vy = m[3] - m[1] * m[1], vxy = m[4] - m[0] * m[1];
      const double S = ((2.0 * m[0] * m[1] + C1) * (2.0 * vxy + C2)) /
                       ((m[0] * m[0] + m[1] * m[1] + C1) * (vx + vy + C2));
      if (y >= kFmR && y < H - kFmR && x >= kFmR && x < W - kFmR) ssim += S;
    }
    __syncthreads();  // hs is rewritten by the next channel
  }
  const double v[kFmStats] = {(double)sse, ssim};  // sse < 2^53: exact
  double* dst = partials + ((size_t)b * gridDim.x + blockIdx.x) * kFmStats;
#pragma unroll
  for (int i = 0; i < kFmStats; ++i) {
    const double r = block_sum(v[i], red);
    if (t == 0) dst[i] = r;
  }
}

// one block per sample: thread t adds partials t, t + 256, ... in order, then the fixed tree; the S sum becomes the mean
__global__ void __launch_bounds__(kMetricsThreads) frame_metrics_sample_kernel(const double* __restrict__ partials,
                                                                               int tiles, double n_crop,
                                                                               double* __restrict__ stats) {
  __shared__ double red[kMetricsThreads];
  const int b = blockIdx.x;
  const double* src = partials + (size_t)b * tiles * kFmStats;
  double v[kFmStats] = {0.0, 0.0};
  for (int c = threadIdx.x; c < tiles; c += kMetricsThreads) {
#pragma unroll
    for (int i = 0; i < kFmStats; ++i) v[i] += src[(size_t)c * kFmStats + i];
  }
  const double sse = block_sum(v[0], red), ssim = block_sum(v[1], red);
  if (threadIdx.x == 0) {
    stats[(size_t)b * kFmStats + 0] = sse;
    stats[(size_t)b * kFmStats + 1] = ssim / n_crop;
  }
}

static size_t frame_metrics_tiles(int H, int W) {
  return (size_t)((W + kFmTileW - 1) / kFmTileW) * (size_t)((H + kFmTileH - 1) / kFmTileH);
}

// ---- F20: label metrics (DAVIS-2017's region similarity J and boundary accuracy F, as integer counts) -----------------
// One block per (kLmTile x kLmTile output tile, frame).  Both label maps are staged with a halo of R = r + 1 (r =
// bound_pix); per object present in the staged labels, the _seg2bmap boundaries of P = (pred == o) and G = (gt == o) are
// computed for the tile plus a halo of r (bit 0: P, bit 1: G; 0 outside the image), then every pixel of the tile adds
// its counts; a boundary pixel searches the disk dx^2 + dy^2 <= r^2 for the other map's boundary.  The block's counts go
// to global memory with one 64-bit integer atomic per (object, count): exact, so the result does not depend on the order.
constexpr int kLmTile = 32;
constexpr int kLmThreads = 256;
constexpr int kLmMaxR = 32;

__device__ __forceinline__ uint8_t lm_bit(const uint8_t* lab, int ls, int r, int c, uint8_t o) {
  return lab[r * ls + c] == o;
}

__global__ void __launch_bounds__(kLmThreads) label_metrics_kernel(const uint8_t* __restrict__ pred,
                                                                   const uint8_t* __restrict__ gt, int H, int W,
                                                                   int tiles_x, int n_objects, int rad,
                                                                   unsigned long long* __restrict__ counts) {
  extern __shared__ uint8_t lm_smem[];
  __shared__ unsigned present[2][8];  // the labels of the staged pred / gt as 256-bit sets
  __shared__ int half[kLmMaxR + 1];   // half[|dy|] = the largest dx with dx^2 + dy^2 <= r^2
  __shared__ unsigned long long red[RB_LABEL_STATS];
  const int t = threadIdx.x, f = blockIdx.y;
  const int R = rad + 1, ls = kLmTile + 2 * R, bs = kLmTile + 2 * rad;
  uint8_t* sp = lm_smem;
  uint8_t* sg = sp + ls * ls;
  uint8_t* bm = sg + ls * ls;
  const int x0 = (int)(blockIdx.x % tiles_x) * kLmTile, y0 = (int)(blockIdx.x / tiles_x) * kLmTile;
  if (t < 16) present[t / 8][t % 8] = 0;
  if (t <= rad) {
    int h = 0;
    while ((h + 1) * (h + 1) + t * t <= rad * rad) ++h;
    half[t] = h;
  }
  __syncthreads();
  const size_t base = (size_t)f * H * W;
  for (int e = t; e < ls * ls; e += kLmThreads) {
    const int y = y0 - R + e / ls, x = x0 - R + e % ls;
    uint8_t p = 0, g = 0;
    if (y >= 0 && y < H && x >= 0 && x < W) {
      p = pred[base + (size_t)y * W + x];
      g = gt[base + (size_t)y * W + x];
      atomicOr(&present[0][p >> 5], 1u << (p & 31));
      atomicOr(&present[1][g >> 5], 1u << (g & 31));
    }
    sp[e] = p;
    sg[e] = g;
  }
  __syncthreads();
  for (int o = 1; o <= n_objects; ++o) {
    if (!((present[0][o >> 5] | present[1][o >> 5]) >> (o & 31) & 1u)) continue;  // the same in every thread
    const uint8_t ob = (uint8_t)o;
    // boundaries of the tile plus a halo of r: b = (m ^ e) | (m ^ s) | (m ^ se), e / s / se 0 outside the image;
    // the last row m ^ e, the last column m ^ s, the last pixel 0
    for (int e = t; e < bs * bs; e += kLmThreads) {
      const int br = e / bs, bc = e % bs, y = y0 - rad + br, x = x0 - rad + bc;
      uint8_t v = 0;
      if (y >= 0 && y < H && x >= 0 && x < W) {
        const int r = br + 1, c = bc + 1;  // in the staged labels
        const bool last_r = y == H - 1, last_c = x == W - 1;
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const uint8_t* lab = k ? sg : sp;
          const uint8_t m = lm_bit(lab, ls, r, c, ob);
          const uint8_t me = last_c ? 0 : lm_bit(lab, ls, r, c + 1, ob);
          const uint8_t ms = last_r ? 0 : lm_bit(lab, ls, r + 1, c, ob);
          const uint8_t mse = (last_r || last_c) ? 0 : lm_bit(lab, ls, r + 1, c + 1, ob);
          uint8_t b;
          if (last_r && last_c) b = 0;
          else if (last_r) b = m ^ me;
          else if (last_c) b = m ^ ms;
          else b = (m ^ me) | (m ^ ms) | (m ^ mse);
          v |= b << k;
        }
      }
      bm[e] = v;
    }
    if (t < RB_LABEL_STATS) red[t] = 0;
    __syncthreads();
    unsigned c[RB_LABEL_STATS] = {0, 0, 0, 0, 0, 0};
    for (int e = t; e < kLmTile * kLmTile; e += kLmThreads) {
      const int i = e / kLmTile, j = e % kLmTile, y = y0 + i, x = x0 + j;
      if (y >= H || x >= W) continue;
      const bool P = sp[(i + R) * ls + j + R] == ob, G = sg[(i + R) * ls + j + R] == ob;
      c[0] += P && G;
      c[1] += P || G;
      const uint8_t v = bm[(i + rad) * bs + j + rad];
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        if (!(v >> k & 1)) continue;
        ++c[2 + k];
        const uint8_t other = (uint8_t)(2 >> k);  // P's boundary looks for G's and G's for P's
        bool hit = false;
        for (int dy = -rad; dy <= rad && !hit; ++dy) {
          const int h = half[dy < 0 ? -dy : dy];
          const uint8_t* row = bm + (i + rad + dy) * bs + j + rad;
          for (int dx = -h; dx <= h; ++dx)
            if (row[dx] & other) {
              hit = true;
              break;
            }
        }
        c[4 + k] += hit;
      }
    }
#pragma unroll
    for (int k = 0; k < RB_LABEL_STATS; ++k) {
      unsigned v = c[k];
      for (int s = 16; s > 0; s >>= 1) v += __shfl_down_sync(0xffffffffu, v, s);
      if ((t & 31) == 0 && v) atomicAdd(&red[k], (unsigned long long)v);
    }
    __syncthreads();
    if (t < RB_LABEL_STATS && red[t]) atomicAdd(&counts[((size_t)f * n_objects + (o - 1)) * RB_LABEL_STATS + t], red[t]);
    __syncthreads();  // bm and red are rewritten by the next object
  }
}

static size_t label_metrics_smem(int rad) {
  const size_t ls = kLmTile + 2 * (rad + 1), bs = kLmTile + 2 * rad;
  return 2 * ls * ls + bs * bs;
}

}  // namespace rb

using namespace rb;

extern "C" int rb_flow_metrics_workspace_bytes(int B, int H, int W, size_t* bytes) {
  RB_REQUIRE(bytes, RB_ERR_BAD_ARG, "rb_flow_metrics_workspace_bytes: null pointer");
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_flow_metrics_workspace_bytes: bad shape B=%d H=%d W=%d", B,
             H, W);
  *bytes = (size_t)B * metrics_chunks(H, W) * kStats * sizeof(double);
  return RB_OK;
}

extern "C" int rb_flow_metrics(const float* flow, float flow_scale, const float* gt, const uint8_t* valid, int B, int H,
                               int W, float* epe, double* stats, void* workspace, size_t workspace_bytes, void* stream) {
  RB_REQUIRE(flow && gt && stats && workspace, RB_ERR_BAD_ARG, "rb_flow_metrics: null pointer");
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_flow_metrics: bad shape B=%d H=%d W=%d", B, H, W);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "rb_flow_metrics: flow_scale must be finite and > 0 (got %g)", (double)flow_scale);
  const size_t npix = (size_t)H * W;
  const size_t chunks = (npix + kMetricsChunk - 1) / kMetricsChunk;
  RB_REQUIRE(B <= 65535 && chunks <= 0x7fffffffu, RB_ERR_BAD_SHAPE,
             "rb_flow_metrics: B=%d samples of %zu pixels exceed one grid", B, npix);
  const size_t need = (size_t)B * chunks * kStats * sizeof(double);
  RB_REQUIRE(workspace_bytes >= need, RB_ERR_WORKSPACE, "rb_flow_metrics: workspace of %zu bytes, %zu needed",
             workspace_bytes, need);
  const cudaStream_t st = (cudaStream_t)stream;
  double* partials = static_cast<double*>(workspace);
  flow_metrics_chunk_kernel<<<dim3((unsigned)chunks, (unsigned)B), kMetricsThreads, 0, st>>>(
      reinterpret_cast<const float2*>(flow), flow_scale, reinterpret_cast<const float2*>(gt), valid, epe, partials, npix);
  RB_CHECK_LAUNCH("flow_metrics_chunk_kernel");
  flow_metrics_sample_kernel<<<B, kMetricsThreads, 0, st>>>(partials, (int)chunks, stats);
  RB_CHECK_LAUNCH("flow_metrics_sample_kernel");
  return RB_OK;
}

extern "C" int rb_frame_metrics_workspace_bytes(int B, int H, int W, size_t* bytes) {
  RB_REQUIRE(bytes, RB_ERR_BAD_ARG, "rb_frame_metrics_workspace_bytes: null pointer");
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_frame_metrics_workspace_bytes: bad shape B=%d H=%d W=%d", B,
             H, W);
  *bytes = (size_t)B * frame_metrics_tiles(H, W) * kFmStats * sizeof(double);
  return RB_OK;
}

extern "C" int rb_frame_metrics(const void* pred, int pred_is_u8, const uint8_t* gt, int B, int H, int W, double* stats,
                                void* workspace, size_t workspace_bytes, void* stream) {
  RB_REQUIRE(pred && gt && stats && workspace, RB_ERR_BAD_ARG, "rb_frame_metrics: null pointer");
  RB_REQUIRE(pred_is_u8 == 0 || pred_is_u8 == 1, RB_ERR_BAD_ARG, "rb_frame_metrics: pred_is_u8 must be 0 or 1 (got %d)",
             pred_is_u8);
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_frame_metrics: bad shape B=%d H=%d W=%d", B, H, W);
  RB_REQUIRE(H >= 2 * kFmR + 1 && W >= 2 * kFmR + 1, RB_ERR_BAD_SHAPE,
             "rb_frame_metrics: H=%d x W=%d is smaller than the 11x11 SSIM window", H, W);
  const size_t tiles = frame_metrics_tiles(H, W);
  RB_REQUIRE(B <= 65535 && tiles <= 0x7fffffffu, RB_ERR_BAD_SHAPE,
             "rb_frame_metrics: B=%d samples of %dx%d pixels exceed one grid", B, H, W);
  const size_t need = (size_t)B * tiles * kFmStats * sizeof(double);
  RB_REQUIRE(workspace_bytes >= need, RB_ERR_WORKSPACE, "rb_frame_metrics: workspace of %zu bytes, %zu needed",
             workspace_bytes, need);
  // scipy's _gaussian_kernel1d(sigma = 1.5, radius 5): exp(-0.5 k^2 / sigma^2), normalised by the sum over k = -5..5
  Gauss11 g;
  double sum = 0.0;
  for (int k = -kFmR; k <= kFmR; ++k) sum += exp(-0.5 * (double)(k * k) / (1.5 * 1.5));
  for (int k = 0; k <= kFmR; ++k) g.w[k] = exp(-0.5 * (double)(k * k) / (1.5 * 1.5)) / sum;
  const cudaStream_t st = (cudaStream_t)stream;
  double* partials = static_cast<double*>(workspace);
  const int tiles_x = (W + kFmTileW - 1) / kFmTileW;
  frame_metrics_tile_kernel<<<dim3((unsigned)tiles, (unsigned)B), kMetricsThreads, 0, st>>>(pred, pred_is_u8, gt, H, W,
                                                                                              tiles_x, g, partials);
  RB_CHECK_LAUNCH("frame_metrics_tile_kernel");
  const double n_crop = 3.0 * (double)(H - 2 * kFmR) * (double)(W - 2 * kFmR);
  frame_metrics_sample_kernel<<<B, kMetricsThreads, 0, st>>>(partials, (int)tiles, n_crop, stats);
  RB_CHECK_LAUNCH("frame_metrics_sample_kernel");
  return RB_OK;
}

extern "C" int rb_label_metrics(const uint8_t* pred, const uint8_t* gt, int n, int H, int W, int n_objects,
                                int bound_pix, int64_t* counts, void* stream) {
  RB_REQUIRE(pred && gt && counts, RB_ERR_BAD_ARG, "rb_label_metrics: null pointer");
  RB_REQUIRE(n > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_label_metrics: bad shape n=%d H=%d W=%d", n, H, W);
  RB_REQUIRE(n_objects >= 1 && n_objects <= 255, RB_ERR_BAD_ARG, "rb_label_metrics: n_objects must be in [1, 255] (got %d)",
             n_objects);
  RB_REQUIRE(bound_pix >= 1 && bound_pix <= kLmMaxR, RB_ERR_BAD_ARG,
             "rb_label_metrics: bound_pix must be in [1, %d] (got %d)", kLmMaxR, bound_pix);
  const size_t tiles = (size_t)((W + kLmTile - 1) / kLmTile) * (size_t)((H + kLmTile - 1) / kLmTile);
  RB_REQUIRE(n <= 65535 && tiles <= 0x7fffffffu, RB_ERR_BAD_SHAPE,
             "rb_label_metrics: n=%d frames of %dx%d pixels exceed one grid", n, H, W);
  const cudaStream_t st = (cudaStream_t)stream;
  RB_CHECK_CUDA(cudaMemsetAsync(counts, 0, (size_t)n * n_objects * RB_LABEL_STATS * sizeof(int64_t), st));
  label_metrics_kernel<<<dim3((unsigned)tiles, (unsigned)n), kLmThreads, label_metrics_smem(bound_pix), st>>>(
      pred, gt, H, W, (W + kLmTile - 1) / kLmTile, n_objects, bound_pix,
      reinterpret_cast<unsigned long long*>(counts));
  RB_CHECK_LAUNCH("label_metrics_kernel");
  return RB_OK;
}
