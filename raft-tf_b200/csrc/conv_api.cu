// A14: stand-alone 'same' convolution with bias (+ReLU), i.e. the tensorpack Conv2D call every hot-path layer is made
// of (stride 1: model_utils.py:112-118,123-128,133-134,142-153,162-166,181-182; stride 2: the encoders' strided layers,
// model_utils.py:21,39,68,92), on fp32 NHWC tensors.  Same kernels as the fused update block: the input is split to fp16 hi/lo planes, the
// HWIO kernel is packed K-major, and the selected back end (wgmma or CUDA-core) runs the implicit
// GEMM.  Used by the parity tests to exercise every filter shape / tile geometry in isolation.
#include <string.h>

#include <vector>

#include "common.cuh"

namespace rb {

static inline size_t align_up_(size_t v, size_t a) { return (v + a - 1) / a * a; }

struct ConvWs {
  __half *in_hi, *in_lo, *w_hi, *w_lo;
  float* bias;
  int cin_pad, cout_pad;
  size_t total;
};

static ConvWs conv_ws_layout(int B, int h, int w, int cin, int cout, int kh, int kw, void* base) {
  ConvWs W;
  char* b = reinterpret_cast<char*>(base);
  W.cin_pad = (cin + 63) / 64 * 64;
  W.cout_pad = (cout + 15) / 16 * 16;
  size_t off = 0;
  auto take = [&](size_t bytes) { char* p = b + off; off += align_up_(bytes, 1024); return p; };
  size_t act = (size_t)B * h * w * W.cin_pad * sizeof(__half);
  size_t wt = (size_t)W.cout_pad * kh * kw * W.cin_pad * sizeof(__half);
  W.in_hi = reinterpret_cast<__half*>(take(act));
  W.in_lo = reinterpret_cast<__half*>(take(act));
  W.w_hi = reinterpret_cast<__half*>(take(wt));
  W.w_lo = reinterpret_cast<__half*>(take(wt));
  W.bias = reinterpret_cast<float*>(take((size_t)W.cout_pad * sizeof(float)));
  W.total = off;
  return W;
}

__global__ void split_pad_kernel(const float* __restrict__ src, __half* __restrict__ hi, __half* __restrict__ lo,
                                 size_t npix, int cin, int cin_pad) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= npix * cin_pad) return;
  size_t pix = i / cin_pad;
  int c = i % cin_pad;
  float v = c < cin ? src[pix * cin + c] : 0.f;
  __half hh, ll;
  split_f32(v, hh, ll);
  hi[i] = hh;
  lo[i] = ll;
}

}  // namespace rb

using namespace rb;

extern "C" int rb_conv2d_workspace_bytes(int B, int h, int w, int cin, int cout, int kh, int kw, size_t* bytes) {
  RB_REQUIRE(bytes && B > 0 && h > 0 && w > 0 && cin > 0 && cout > 0 && kh > 0 && kw > 0, RB_ERR_BAD_ARG,
             "rb_conv2d_workspace_bytes: bad argument");
  *bytes = conv_ws_layout(B, h, w, cin, cout, kh, kw, nullptr).total;
  return RB_OK;
}

extern "C" int rb_conv2d(const float* x, const float* W_host, const float* b_host, float* y, int B, int h, int w,
                         int cin, int cout, int kh, int kw, int relu, void* workspace, size_t workspace_bytes,
                         void* stream) {
  return rb_conv2d_strided(x, W_host, b_host, y, B, h, w, cin, cout, kh, kw, 1, relu, workspace, workspace_bytes, stream);
}

extern "C" int rb_conv2d_strided(const float* x, const float* W_host, const float* b_host, float* y, int B, int h, int w,
                                 int cin, int cout, int kh, int kw, int stride, int relu, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  RB_REQUIRE(x && W_host && y && workspace, RB_ERR_BAD_ARG, "rb_conv2d: null pointer");
  RB_REQUIRE(B > 0 && h > 0 && w > 0 && cin > 0 && cout > 0, RB_ERR_BAD_SHAPE, "rb_conv2d: bad shape");
  RB_REQUIRE((kh & 1) && (kw & 1) && kh <= 7 && kw <= 7, RB_ERR_UNSUPPORTED,
             "rb_conv2d: only odd kernels up to 7 ('same'), got %dx%d", kh, kw);
  RB_REQUIRE(stride == 1 || stride == 2, RB_ERR_UNSUPPORTED, "rb_conv2d: stride %d (1 and 2 are what the reference uses)", stride);
  ConvWs L = conv_ws_layout(B, h, w, cin, cout, kh, kw, workspace);
  RB_REQUIRE(workspace_bytes >= L.total, RB_ERR_WORKSPACE, "rb_conv2d: workspace has %zu bytes, need %zu", workspace_bytes,
             L.total);
  cudaStream_t s = (cudaStream_t)stream;
  const int taps = kh * kw;
  // pack weights on the host: HWIO -> [cout_pad][tap][cin_pad] split planes
  size_t welems = (size_t)L.cout_pad * taps * L.cin_pad;
  std::vector<__half> hi(welems, __float2half_rn(0.f)), lo(welems, __float2half_rn(0.f));
  std::vector<float> bias(L.cout_pad, 0.f);
  for (int t = 0; t < taps; ++t)
    for (int ci = 0; ci < cin; ++ci)
      for (int co = 0; co < cout; ++co) {
        size_t o = ((size_t)co * taps + t) * L.cin_pad + ci;
        split_f32(W_host[((size_t)t * cin + ci) * cout + co], hi[o], lo[o]);
      }
  if (b_host) memcpy(bias.data(), b_host, (size_t)cout * sizeof(float));
  RB_CHECK_CUDA(cudaMemcpyAsync(L.w_hi, hi.data(), welems * sizeof(__half), cudaMemcpyHostToDevice, s));
  RB_CHECK_CUDA(cudaMemcpyAsync(L.w_lo, lo.data(), welems * sizeof(__half), cudaMemcpyHostToDevice, s));
  RB_CHECK_CUDA(cudaMemcpyAsync(L.bias, bias.data(), (size_t)L.cout_pad * sizeof(float), cudaMemcpyHostToDevice, s));
  RB_CHECK_CUDA(cudaStreamSynchronize(s));
  size_t npix = (size_t)B * h * w;
  size_t n = npix * L.cin_pad;
  split_pad_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(x, L.in_hi, L.in_lo, npix, cin, L.cin_pad);
  RB_CHECK_LAUNCH("split_pad_kernel");
  ConvParams p;
  memset(&p, 0, sizeof(p));
  p.in_hi = L.in_hi; p.in_lo = L.in_lo; p.in_stride = L.cin_pad; p.in_choff = 0; p.cin_pad = L.cin_pad;
  p.w_hi = L.w_hi; p.w_lo = L.w_lo; p.bias = L.bias;
  p.cout = cout; p.cout_pad = L.cout_pad; p.kh = kh; p.kw = kw;
  p.B = B; p.h = h; p.w = w;
  if (stride != 1) {  // strided input view (ConvParams, common.cuh): y is [B, ceil(h/s), ceil(w/s), cout]
    int pt, pl, oh, ow;
    conv_pad_before(h, kh, stride, semantics(), &pt, &oh);
    conv_pad_before(w, kw, stride, semantics(), &pl, &ow);
    p.in_h = h; p.in_w = w; p.h = oh; p.w = ow;
    p.sx = p.sy = stride;
    p.pad_explicit = 1; p.pad_x = pl; p.pad_y = pt;
  }
  p.epi = EPI_F32; p.act = relu ? ACT_RELU : ACT_NONE; p.scale = 1.f; p.f0 = y;
  return launch_conv(p, s);
}
