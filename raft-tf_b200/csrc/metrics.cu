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
