// A13: flow upsampling.  Reference: RAFT.upsample_flow (networks/RAFT.py:119-134) and upflow8
// (networks/utils.py:105-111).
#include "common.cuh"

namespace rb {

// Convex 8x upsampling.  One thread per fine pixel (sy,sx) of a coarse pixel; 4 coarse pixels per
// block.  mask channel = k*64 + sy*8 + sx with k = ky*3+kx (RAFT.py:125); softmax over k (:126);
// 3x3 zero-padded patches of 8*flow (:128); weighted sum over k (:131).
// The output may be a CROP of the 8h x 8w field: out is [B,oH,oW,2] and holds rows [top, top+oH) x cols [left, left+oW)
// (frames that were replicate-padded to a multiple of 8 are cropped back here, not by a torch slice afterwards).
__global__ void __launch_bounds__(256) upsample_convex_kernel(const float2* __restrict__ coords1,
                                                              const float* __restrict__ mask,
                                                              float2* __restrict__ out, int B, int h, int w, int top,
                                                              int left, int oH, int oW) {
  const int cp = blockIdx.x * 4 + (threadIdx.x >> 6);
  const int t = threadIdx.x & 63;
  if (cp >= B * h * w) return;
  const int x = cp % w, y = (cp / w) % h, b = cp / (w * h);
  const float* m = mask + (size_t)cp * 576 + t;
  float v[9];
  float mx = -INFINITY;
#pragma unroll
  for (int k = 0; k < 9; ++k) { v[k] = m[k * 64]; mx = fmaxf(mx, v[k]); }
  float sum = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) { v[k] = expf(v[k] - mx); sum += v[k]; }
  float ax = 0.f, ay = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
    float fx = 0.f, fy = 0.f;
    if (yy >= 0 && yy < h && xx >= 0 && xx < w) {
      float2 c = coords1[(size_t)(b * h + yy) * w + xx];
      fx = 8.0f * (c.x - (float)xx);
      fy = 8.0f * (c.y - (float)yy);
    }
    const float p = v[k] / sum;  // IEEE quotient
    ax = __fmaf_rn(fx, p, ax);
    ay = __fmaf_rn(fy, p, ay);
  }
  const int oy = y * 8 + (t >> 3) - top, ox = x * 8 + (t & 7) - left;
  if (oy >= 0 && oy < oH && ox >= 0 && ox < oW) out[((size_t)b * oH + oy) * oW + ox] = make_float2(ax, ay);
}

// tf.image.resize_bilinear(flow, 8x, align_corners=True) -- and no x8 of the values unless
// scale says so (reference quirk, utils.py:110).
__global__ void upflow8_kernel(const float2* __restrict__ coords1, float2* __restrict__ out, int B, int h, int w,
                               float scale, int top, int left, int oH, int oW) {
  const int H = 8 * h, Wd = 8 * w;
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * oH * oW) return;
  const int ox = (int)(i % oW) + left, oy = (int)((i / oW) % oH) + top, b = (int)(i / ((size_t)oW * oH));
  const float sy = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f;
  const float sx = Wd > 1 ? (float)(w - 1) / (float)(Wd - 1) : 0.f;
  const float fy = (float)oy * sy, fx = (float)ox * sx;
  const int y0 = (int)floorf(fy), x0 = (int)floorf(fx);
  const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
  const float ly = fy - (float)y0, lx = fx - (float)x0;
  auto flow = [&](int yy, int xx) {
    float2 c = coords1[(size_t)(b * h + yy) * w + xx];
    return make_float2(c.x - (float)xx, c.y - (float)yy);
  };
  const float2 tl = flow(y0, x0), tr = flow(y0, x1), bl = flow(y1, x0), br = flow(y1, x1);
  const float topx = tl.x + (tr.x - tl.x) * lx, topy = tl.y + (tr.y - tl.y) * lx;
  const float botx = bl.x + (br.x - bl.x) * lx, boty = bl.y + (br.y - bl.y) * lx;
  out[i] = make_float2(scale * (topx + (botx - topx) * ly), scale * (topy + (boty - topy) * ly));
}

}  // namespace rb

using namespace rb;

static int check_crop(const char* fn, int h, int w, int top, int left, int oH, int oW) {
  RB_REQUIRE(top >= 0 && left >= 0 && oH > 0 && oW > 0 && top + oH <= 8 * h && left + oW <= 8 * w, RB_ERR_BAD_SHAPE,
             "%s: crop rows [%d,%d) cols [%d,%d) outside the %dx%d field", fn, top, top + oH, left, left + oW, 8 * h, 8 * w);
  return RB_OK;
}

extern "C" int rb_upsample_convex_crop(const float* coords1, const float* mask, float* out, int B, int h, int w, int top,
                                       int left, int out_h, int out_w, void* stream) {
  RB_REQUIRE(coords1 && mask && out, RB_ERR_BAD_ARG, "rb_upsample_convex: null pointer");
  RB_REQUIRE(B > 0 && h > 0 && w > 0, RB_ERR_BAD_SHAPE, "rb_upsample_convex: bad shape");
  int rc = check_crop("rb_upsample_convex_crop", h, w, top, left, out_h, out_w);
  if (rc) return rc;
  int n = B * h * w;
  upsample_convex_kernel<<<(n + 3) / 4, 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float2*>(coords1), mask, reinterpret_cast<float2*>(out), B, h, w, top, left, out_h, out_w);
  RB_CHECK_LAUNCH("upsample_convex_kernel");
  return RB_OK;
}

extern "C" int rb_upsample_convex(const float* coords1, const float* mask, float* out, int B, int h, int w,
                                  void* stream) {
  return rb_upsample_convex_crop(coords1, mask, out, B, h, w, 0, 0, 8 * h, 8 * w, stream);
}

extern "C" int rb_upflow8_crop(const float* coords1, float* out, int B, int h, int w, float scale, int top, int left,
                               int out_h, int out_w, void* stream) {
  RB_REQUIRE(coords1 && out, RB_ERR_BAD_ARG, "rb_upflow8: null pointer");
  RB_REQUIRE(B > 0 && h > 0 && w > 0, RB_ERR_BAD_SHAPE, "rb_upflow8: bad shape");
  int rc = check_crop("rb_upflow8_crop", h, w, top, left, out_h, out_w);
  if (rc) return rc;
  size_t n = (size_t)B * out_h * out_w;
  upflow8_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float2*>(coords1), reinterpret_cast<float2*>(out), B, h, w, scale, top, left, out_h, out_w);
  RB_CHECK_LAUNCH("upflow8_kernel");
  return RB_OK;
}

extern "C" int rb_upflow8(const float* coords1, float* out, int B, int h, int w, float scale, void* stream) {
  return rb_upflow8_crop(coords1, out, B, h, w, scale, 0, 0, 8 * h, 8 * w, stream);
}
