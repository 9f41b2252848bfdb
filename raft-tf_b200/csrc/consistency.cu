// F5: forward-backward consistency of a bidirectional flow pair (Sundaram et al. 2010; UnFlow, Meister et al. 2018).
// The reference estimates flow 1->0 by splatting flow 0->1 (flow_utils.py:166 reverse_flow_avg_skip_static) and computes no
// occlusion mask; this is the standard check on two real flows, used by frame interpolation to find occluded pixels.
#include <math.h>

#include "common.cuh"
#include "fb_sample.cuh"

namespace rb {

// One thread per (direction, pixel); threads [0, npix) check fw against bw, [npix, 2 npix) bw against fw.
// Every operation is rounded on its own, left to right (__fmul_rn/__fadd_rn: no FMA contraction), so the mask is reproduced
// bit for bit by an fp32 restatement -- a pixel near the threshold does not flip between implementations.
__global__ void __launch_bounds__(256) flow_fb_check_kernel(const float2* __restrict__ flow_fw,
                                                            const float2* __restrict__ flow_bw,
                                                            uint8_t* __restrict__ occ_fw, uint8_t* __restrict__ occ_bw,
                                                            int H, int W, size_t npix, float s, float a1, float a2) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= 2 * npix) return;
  const bool back = i >= npix;
  const size_t p = back ? i - npix : i;
  const float2* __restrict__ fsrc = back ? flow_bw : flow_fw;
  const float2* __restrict__ bsrc = back ? flow_fw : flow_bw;
  uint8_t* __restrict__ out = back ? occ_bw : occ_fw;
  const int x = (int)(p % W), y = (int)((p / W) % H);
  const size_t img = p - ((size_t)y * W + x);  // first pixel of this sample
  const float2 fr = fsrc[p];
  const float2 f = make_float2(__fmul_rn(s, fr.x), __fmul_rn(s, fr.y));
  const float qx = __fadd_rn((float)x, f.x), qy = __fadd_rn((float)y, f.y);
  if (!inside_frame(qx, qy, H, W)) {
    out[p] = 2;
    return;
  }
  const float2 b = sample_flow(bsrc + img, W, bilerp_at(qx, qy, H, W), s);
  out[p] = fb_inconsistent(f, b, a1, a2);
}

}  // namespace rb

using namespace rb;

extern "C" int rb_flow_fb_check(const float* flow_fw, const float* flow_bw, uint8_t* occ_fw, uint8_t* occ_bw, int B, int H,
                                int W, float flow_scale, float alpha1, float alpha2, void* stream) {
  RB_REQUIRE(flow_fw && flow_bw && occ_fw && occ_bw, RB_ERR_BAD_ARG, "rb_flow_fb_check: null pointer");
  RB_REQUIRE(B > 0 && H > 0 && W > 0, RB_ERR_BAD_SHAPE, "rb_flow_fb_check: bad shape B=%d H=%d W=%d", B, H, W);
  RB_REQUIRE(flow_scale > 0.f && isfinite(flow_scale), RB_ERR_BAD_ARG,
             "rb_flow_fb_check: flow_scale must be finite and > 0 (got %g)", (double)flow_scale);
  RB_REQUIRE(alpha1 >= 0.f && isfinite(alpha1) && alpha2 >= 0.f && isfinite(alpha2), RB_ERR_BAD_ARG,
             "rb_flow_fb_check: alpha1, alpha2 must be finite and >= 0 (got %g, %g)", (double)alpha1, (double)alpha2);
  const size_t npix = (size_t)B * H * W;
  const size_t blocks = (2 * npix + 255) / 256;
  RB_REQUIRE(blocks <= 0x7fffffffu, RB_ERR_BAD_SHAPE, "rb_flow_fb_check: %zu pixels exceed one grid", npix);
  flow_fb_check_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      reinterpret_cast<const float2*>(flow_fw), reinterpret_cast<const float2*>(flow_bw), occ_fw, occ_bw, H, W, npix,
      flow_scale, alpha1, alpha2);
  RB_CHECK_LAUNCH("flow_fb_check_kernel");
  return RB_OK;
}
