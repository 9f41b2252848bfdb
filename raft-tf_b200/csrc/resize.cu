// F3 (input/output edge): the bilinear cv2.resize the reference applies to every frame (dataflow/test_dataflow.py:85-87,
// to 432x1024) and to flows (flow_utils.py:277-284 resize_flow), bit for bit with OpenCV 4.13 as the reference's
// environment ships it.  cv2 runs two algorithms (tests/resize_oracle.py restates both):
//   uint8:   OpenCV's fixed-point code -- fp32 coordinates, 11-bit coefficients, the SIMD path's vertical rounding;
//   float32: Intel IPP's linear resize (float64 coordinates, fmaf(w, p1 - p0, p0) per pass), except for a single-row
//            or single-column source, where cv2 runs OpenCV's own float code; a same-size resize is a copy.
// One thread per output pixel evaluates both passes on the fly (4 taps, coefficients computed in-kernel with explicitly
// rounded operations, so no FMA contraction changes them).
#include <climits>

#include "resize_px.cuh"

namespace rb {

// uint8 resize of pixel (y, x) of one channel-interleaved [H,W,C] plane; returns the 0..255 value per channel
template <int C>
__device__ __forceinline__ void resize_u8_px(const uint8_t* __restrict__ p, int H, int W, int Ho, int Wo, int y, int x,
                                             int out[C]) {
  int sx, sy;
  float fx, fy;
  cv_coord(x, 1.0 / ((double)Wo / W), sx, fx);
  cv_coord(y, 1.0 / ((double)Ho / H), sy, fy);
  if (sx < 0) { sx = 0; fx = 0.f; }  // horizontally the fraction of a clamped column is dropped ...
  if (sx >= W - 1) { sx = W - 1; fx = 0.f; }
  const int x0 = sx, x1 = min(sx + 1, W - 1);
  const int y0 = min(max(sy, 0), H - 1), y1 = min(max(sy + 1, 0), H - 1);  // ... vertically only the row is clamped
  const int a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fx), 2048.f)), a1 = __float2int_rn(__fmul_rn(fx, 2048.f));
  const int b0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, fy), 2048.f)), b1 = __float2int_rn(__fmul_rn(fy, 2048.f));
  const uint8_t *r0 = p + (size_t)y0 * W * C, *r1 = p + (size_t)y1 * W * C;
#pragma unroll
  for (int c = 0; c < C; ++c) {
    const int s0 = r0[x0 * C + c] * a0 + r0[x1 * C + c] * a1;
    const int s1 = r1[x0 * C + c] * a0 + r1[x1 * C + c] * a1;
    // OpenCV's SIMD vertical pass: 16-bit high products of the coefficients and S >> 4, then (sum + 2) >> 2
    const int v = (((b0 * (s0 >> 4)) >> 16) + ((b1 * (s1 >> 4)) >> 16) + 2) >> 2;
    out[c] = min(max(v, 0), 255);
  }
}

// dst [B,Hp,Wp,3] fp32 in [0,1]: the Ho x Wo resize of src [B,H,W,3], replicate-padded by (pad_top, pad_left, ...)
template <bool U8>
__global__ void frames_resize_kernel(const void* __restrict__ src, float* __restrict__ dst, int B, int H, int W, int Ho,
                                     int Wo, int Hp, int Wp, int pad_top, int pad_left, int mode) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * Hp * Wp) return;
  const int xp = (int)(i % Wp), yp = (int)((i / Wp) % Hp), b = (int)(i / ((size_t)Wp * Hp));
  const int x = min(max(xp - pad_left, 0), Wo - 1), y = min(max(yp - pad_top, 0), Ho - 1);  // pad after the resize
  float v[3];
  if (U8) {
    int u[3];
    resize_u8_px<3>(reinterpret_cast<const uint8_t*>(src) + (size_t)b * H * W * 3, H, W, Ho, Wo, y, x, u);
#pragma unroll
    for (int c = 0; c < 3; ++c) v[c] = __fdiv_rn((float)u[c], 255.0f);  // np.float32(x) / 255.0, as rb_frames_prepare
  } else {
    resize_f32_px<3>(reinterpret_cast<const float*>(src) + (size_t)b * H * W * 3, H, W, Ho, Wo, y, x, mode, v);
  }
  float* d = dst + i * 3;
  d[0] = v[0]; d[1] = v[1]; d[2] = v[2];
}

// dst [B,Ho,Wo,2]: both channels of flow [B,H,W,2] resized, then u *= su, v *= sv (flow_utils.py:280-281)
__global__ void flow_resize_kernel(const float* __restrict__ flow, float* __restrict__ dst, int B, int H, int W, int Ho,
                                   int Wo, int mode, float su, float sv) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * Ho * Wo) return;
  const int x = (int)(i % Wo), y = (int)((i / Wo) % Ho), b = (int)(i / ((size_t)Wo * Ho));
  float v[2];
  resize_f32_px<2>(flow + (size_t)b * H * W * 2, H, W, Ho, Wo, y, x, mode, v);
  dst[i * 2] = __fmul_rn(v[0], su);
  dst[i * 2 + 1] = __fmul_rn(v[1], sv);
}

}  // namespace rb

using namespace rb;

extern "C" int rb_frames_resize(const void* src, int src_is_u8, float* dst, int B, int H, int W, int Ho, int Wo,
                                int pad_top, int pad_bottom, int pad_left, int pad_right, void* stream) {
  RB_REQUIRE(src && dst, RB_ERR_BAD_ARG, "rb_frames_resize: null pointer");
  RB_REQUIRE(B > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0 && pad_top >= 0 && pad_bottom >= 0 && pad_left >= 0 &&
                 pad_right >= 0,
             RB_ERR_BAD_SHAPE, "rb_frames_resize: bad shape B=%d H=%d W=%d Ho=%d Wo=%d pad=(%d,%d,%d,%d)", B, H, W, Ho, Wo,
             pad_top, pad_bottom, pad_left, pad_right);
  const long long Hp = (long long)Ho + pad_top + pad_bottom, Wp = (long long)Wo + pad_left + pad_right;
  RB_REQUIRE(Hp <= INT_MAX && Wp <= INT_MAX && (long long)H * W * 3 <= INT_MAX, RB_ERR_BAD_SHAPE,
             "rb_frames_resize: frame too large (%d x %d -> %lld x %lld)", H, W, Hp, Wp);
  const size_t n = (size_t)B * Hp * Wp;
  const unsigned blocks = (unsigned)((n + 255) / 256);
  if (src_is_u8)
    frames_resize_kernel<true><<<blocks, 256, 0, (cudaStream_t)stream>>>(src, dst, B, H, W, Ho, Wo, (int)Hp, (int)Wp,
                                                                         pad_top, pad_left, RS_COPY);
  else
    frames_resize_kernel<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(src, dst, B, H, W, Ho, Wo, (int)Hp, (int)Wp,
                                                                          pad_top, pad_left, float_mode(H, W, Ho, Wo));
  RB_CHECK_LAUNCH("frames_resize_kernel");
  return RB_OK;
}

extern "C" int rb_flow_resize(const float* flow, float* dst, int B, int H, int W, int Ho, int Wo, void* stream) {
  RB_REQUIRE(flow && dst, RB_ERR_BAD_ARG, "rb_flow_resize: null pointer");
  RB_REQUIRE(B > 0 && H > 0 && W > 0 && Ho > 0 && Wo > 0, RB_ERR_BAD_SHAPE,
             "rb_flow_resize: bad shape B=%d H=%d W=%d Ho=%d Wo=%d", B, H, W, Ho, Wo);
  RB_REQUIRE((long long)H * W * 2 <= INT_MAX && (long long)Ho * Wo * 2 <= INT_MAX, RB_ERR_BAD_SHAPE,
             "rb_flow_resize: flow too large (%d x %d -> %d x %d)", H, W, Ho, Wo);
  const float su = flow_scale_u(W, Wo), sv = flow_scale_v(H, Ho);
  const size_t n = (size_t)B * Ho * Wo;
  flow_resize_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(flow, dst, B, H, W, Ho, Wo,
                                                                                    float_mode(H, W, Ho, Wo), su, sv);
  RB_CHECK_LAUNCH("flow_resize_kernel");
  return RB_OK;
}
