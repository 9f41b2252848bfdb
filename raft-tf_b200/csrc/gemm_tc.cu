// A1 on tensor cores: the all-pairs correlation volume and its pyramid as four GEMMs.
// Reference: networks/model_utils.py:199-221 (GetCorrPyramid).
//
// level 0:  vol0[n, m] = <fmap1[n,:], fmap2[m,:]> / sqrt(C)
// level l:  the reference average-pools the h2 x w2 axes of the volume (2x2, stride 2, VALID).
//           Pooling is linear, so  pool(vol)[n, m'] = <fmap1[n,:], pool(fmap2)[m',:]> / sqrt(C):
//           instead of re-reading the 4*N^2-byte volume three times we pool the (tiny) fmap2 and
//           run three more GEMMs (+33% MMA work, no extra HBM reads).  Identical in exact
//           arithmetic; differs from pooling the stored fp32 volume by fp32 rounding only
//           (tests/test_gpu_fullsize.py::test_pyramid_levels_are_valid_avgpools_fullsize, tests/test_oracle.py::test_pool_linearity_valid_floor).
// The GEMMs reuse the implicit-GEMM kernel of conv_tc.cu with a 1x1 "filter" whose weight operand
// is the (pooled) fmap2 of the same batch element.
#include <math.h>
#include <string.h>

#include "packed.cuh"

namespace rb {

struct CorrWs {
  SplitPtr f1;
  SplitPtr f2[RB_NUM_LEVELS];
  size_t total;
};

// rows of pyramid level l, padded to a multiple of 16 so the "weight" operand has a legal cout_pad
static int level_rows(int h, int w, int l) { return level_dim(h, l) * level_dim(w, l); }
static int level_rows_pad(int h, int w, int l) { return round_up(level_rows(h, w, l), 16); }

static CorrWs corr_ws_layout(int B, int h, int w, int C, void* base) {
  CorrWs W;
  Arena a(base);
  W.f1 = a.split((size_t)B * h * w * C);
  for (int l = 0; l < RB_NUM_LEVELS; ++l) W.f2[l] = a.split((size_t)B * level_rows_pad(h, w, l) * C);
  W.total = a.size;
  return W;
}

size_t corr_tc_workspace_bytes(int B, int h, int w, int C) { return corr_ws_layout(B, h, w, C, nullptr).total; }

// ONE preparation launch (seven separate split / pool launches with one element per thread took a third of the build).
// blockIdx.y selects the section:
//   0: fmap1 -> split planes            1: fmap2 -> split planes (pyramid level 0)
//   2..4: pool^l(fmap2) -> split planes, l = 1..3, evaluated hierarchically from fmap2 itself with exactly the rounding of
//         l successive 2x2 VALID average pools ((a+b+c+d)*0.25 per stage, model_utils.py:217-219 by linearity)
// 4 channels per thread (float4 in, 8-byte stores per plane); rows in [rows, rows_pad) are zero.
template <int L>
__device__ __forceinline__ float4 pooled_px(const float* __restrict__ f2, int W0, int C, int y, int x, int c) {
  if constexpr (L == 0) {
    return __ldg(reinterpret_cast<const float4*>(f2 + ((size_t)y * W0 + x) * C + c));
  } else {
    const float4 a = pooled_px<L - 1>(f2, W0, C, 2 * y, 2 * x, c), b = pooled_px<L - 1>(f2, W0, C, 2 * y, 2 * x + 1, c);
    const float4 d = pooled_px<L - 1>(f2, W0, C, 2 * y + 1, 2 * x, c), e = pooled_px<L - 1>(f2, W0, C, 2 * y + 1, 2 * x + 1, c);
    return make_float4((a.x + b.x + d.x + e.x) * 0.25f, (a.y + b.y + d.y + e.y) * 0.25f, (a.z + b.z + d.z + e.z) * 0.25f,
                       (a.w + b.w + d.w + e.w) * 0.25f);
  }
}
struct CorrPrep {
  const float* f1;
  const float* f2;
  __half* hi[5];
  __half* lo[5];
  int rows[5], rows_pad[5], wl[5];  // per section: valid rows per sample, padded rows, level width
  int B, h, w, C;
};
__global__ void __launch_bounds__(256) corr_prep_kernel(const CorrPrep P) {
  const int sec = blockIdx.y;
  const int c4 = P.C / 4;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t per = (size_t)P.rows_pad[sec] * c4;
  if (i >= (size_t)P.B * per) return;
  const int b = (int)(i / per);
  const size_t rem = i - (size_t)b * per;
  const int r = (int)(rem / c4), c = (int)(rem % c4) * 4;
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (r < P.rows[sec]) {
    const size_t N0 = (size_t)P.h * P.w;
    if (sec == 0) {
      v = __ldg(reinterpret_cast<const float4*>(P.f1 + ((size_t)b * N0 + r) * P.C + c));
    } else {
      const float* f2 = P.f2 + (size_t)b * N0 * P.C;
      const int y = r / P.wl[sec], x = r - y * P.wl[sec];
      if (sec == 1) v = pooled_px<0>(f2, P.w, P.C, y, x, c);
      else if (sec == 2) v = pooled_px<1>(f2, P.w, P.C, y, x, c);
      else if (sec == 3) v = pooled_px<2>(f2, P.w, P.C, y, x, c);
      else v = pooled_px<3>(f2, P.w, P.C, y, x, c);
    }
  }
  uint32_t h0, l0, h1, l1;
  split2(v.x, v.y, h0, l0);
  split2(v.z, v.w, h1, l1);
  const size_t o = ((size_t)b * P.rows_pad[sec] + r) * P.C + c;
  *reinterpret_cast<uint2*>(P.hi[sec] + o) = make_uint2(h0, h1);
  *reinterpret_cast<uint2*>(P.lo[sec] + o) = make_uint2(l0, l1);
}

int corr_build_tc(const float* fmap1, const float* fmap2, float* pyramid, int B, int h, int w, int C, void* ws,
                  size_t ws_bytes, cudaStream_t s) {
  RB_REQUIRE(C % 64 == 0, RB_ERR_BAD_SHAPE, "rb_corr_build (tensor-core): C=%d must be a multiple of 64", C);
  size_t need = corr_tc_workspace_bytes(B, h, w, C);
  RB_REQUIRE(ws && ws_bytes >= need, RB_ERR_WORKSPACE, "rb_corr_build: workspace has %zu bytes, need %zu", ws_bytes, need);
  CorrWs W = corr_ws_layout(B, h, w, C, ws);
  const int N = h * w;
  {
    CorrPrep P;
    memset(&P, 0, sizeof(P));
    P.f1 = fmap1; P.f2 = fmap2; P.B = B; P.h = h; P.w = w; P.C = C;
    P.hi[0] = W.f1.hi; P.lo[0] = W.f1.lo; P.rows[0] = N; P.rows_pad[0] = N; P.wl[0] = w;
    size_t max_items = (size_t)B * N * (C / 4);
    for (int l = 0; l < RB_NUM_LEVELS; ++l) {
      P.hi[l + 1] = W.f2[l].hi; P.lo[l + 1] = W.f2[l].lo;
      P.rows[l + 1] = level_rows(h, w, l); P.rows_pad[l + 1] = level_rows_pad(h, w, l); P.wl[l + 1] = level_dim(w, l);
      const size_t items = (size_t)B * P.rows_pad[l + 1] * (C / 4);
      if (items > max_items) max_items = items;
    }
    dim3 grid((unsigned)((max_items + 255) / 256), 5);
    corr_prep_kernel<<<grid, 256, 0, s>>>(P);
    RB_CHECK_LAUNCH("corr_prep_kernel");
  }
  size_t lvl_off = 0;
  for (int l = 0; l < RB_NUM_LEVELS; ++l) {
    const int rows = level_rows(h, w, l);
    // the (pooled) fmap2 of each batch element as the 1x1 "filter": rows = output channels, C = input channels
    const ConvWeights f2 = {W.f2[l].hi, W.f2[l].lo, nullptr, 1, 1, C, rows, level_rows_pad(h, w, l)};
    ConvParams p = conv_params(f2, W.f1, C, 0, B, h, w);
    p.w_per_batch = 1;
    p.epi = EPI_F32;
    {  // divide after the matmul (:213).  sqrt(256) = 16: the division is an exact scaling, a multiply gives the same bits
      const float sq = sqrtf((float)C);
      int e;
      const bool pow2 = frexpf(sq, &e) == 0.5f;
      p.scale = (float)(1.0 / (double)sq);  // the divisor's reciprocal, rounded once (div_rn in common.cuh)
      p.div = pow2 ? 0.f : sq;
    }
    p.f0 = pyramid + lvl_off;
    int rc = launch_conv_tc(p, s);
    if (rc) return rc;
    lvl_off += (size_t)B * N * rows;
  }
  return RB_OK;
}

}  // namespace rb
